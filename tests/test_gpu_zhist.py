"""RedshiftHistogram on the GPU against the restatement of oracle/zhist_oracle.py: Scott's edges to 1e-13, counts exactly
on the device's own edges and weighted sums to 1e-12 of sum |w| per bin, for Scott's rule, int bins, even and non-uniform
explicit edges, float32 / float64 redshifts and weights, rows on every edge, both sides of the shared-memory / global
histogram choice and 1- and 2-row catalogues; the reference tests' assertions (test_unweighted, test_weighted,
test_save); `interpolate` against scipy in all four extrapolation modes; the golden fixtures of the reference's output;
P = 2 and 3 processes over gloo sharing device 0; and the reference's test_with_zhist through ConvolvedFFTPower.
tests/mgpu_check_zhist.py runs the several-rank comparison under torchrun on several GPUs."""
import datetime
import os
import socket
import sys
import warnings

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import zhist_oracle as zo

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
FSKY = 0.15


def _cosmo():
    from nbodykit_b200.cosmology import Planck15
    return Planck15


def _cat(z, w=None, comm=None, device=True):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ArrayCatalog
    cols = {"z": torch.from_numpy(np.ascontiguousarray(z)).cuda() if device else np.ascontiguousarray(z)}
    if w is not None:
        cols["w"] = torch.from_numpy(np.ascontiguousarray(w)).cuda() if device else np.ascontiguousarray(w)
    return ArrayCatalog(cols, comm=comm or SelfComm())


def _run(z, w=None, bins=None, comm=None, device=True):
    from nbodykit_b200.lab import RedshiftHistogram
    return RedshiftHistogram(_cat(z, w, comm, device), FSKY, _cosmo(), bins=bins, redshift="z",
                             weight="w" if w is not None else None)


def _check(z, w=None, bins=None):
    """the device result against the oracle: edges to 1e-13, counts exact on the device's edges, sums to 1e-12 sum |w|"""
    r = _run(z, w, bins)
    if bins is None:
        want = zo.scott_edges(z)[1]
        assert len(r.bin_edges) == len(want)
        np.testing.assert_allclose(r.bin_edges, want, rtol=1e-13, atol=0)
    elif np.isscalar(bins):
        np.testing.assert_array_equal(r.bin_edges, zo.int_edges(z, bins))
    else:
        np.testing.assert_array_equal(r.bin_edges, np.asarray(bins, "f8"))
    dV = zo.shell_volumes(r.bin_edges, FSKY, _cosmo())
    np.testing.assert_array_equal(r.dV, dV)
    np.testing.assert_array_equal(r.bin_centers, 0.5 * (r.bin_edges[1:] + r.bin_edges[:-1]))
    if w is None:
        np.testing.assert_array_equal(r.nbar * 1.0, zo.counts(z, r.bin_edges) / dV)
        np.testing.assert_array_equal(np.rint(r.nbar * dV), zo.counts(z, r.bin_edges))
    else:
        want = zo.counts(z, r.bin_edges, w)
        absw = zo.counts(z, r.bin_edges, np.abs(np.asarray(w, "f8")))
        assert (np.abs(r.nbar * dV - want) <= 1e-12 * absw + 1e-300).all()
    return r


@pytest.mark.parametrize("zdt", ["f4", "f8"])
@pytest.mark.parametrize("wdt", [None, "f4", "f8"])
@pytest.mark.parametrize("n", [1000, 200000])
def test_scott(cuda, n, zdt, wdt):
    z = zo.make_redshifts(42, n).astype(zdt)
    w = None if wdt is None else np.random.RandomState(1).uniform(-0.5, 1.5, n).astype(wdt)
    _check(z, w)


@pytest.mark.parametrize("bins", [1, 7, 50])
@pytest.mark.parametrize("zdt", ["f4", "f8"])
def test_int_bins(cuda, bins, zdt):
    z = zo.make_redshifts(3, 5000).astype(zdt)
    r = _check(z, None, bins)
    # the row at the maximum sits on the last edge and is not counted
    assert np.rint(r.nbar * r.dV).sum() == (z.astype("f8") < z.max()).sum()


def _edges(kind, nb):
    if kind == "even":
        return np.linspace(0.05, 1.05, nb + 1)
    # non-uniform: growing widths
    e = 0.05 + np.cumsum(np.r_[0.0, np.random.RandomState(nb).uniform(0.2, 1.8, nb)])
    return 0.05 + (e - 0.05) / (e[-1] - 0.05)


@pytest.mark.parametrize("kind", ["even", "nonuniform"])
@pytest.mark.parametrize("nb", [200, 4096, 4097, 12000])
@pytest.mark.parametrize("wdt", [None, "f4", "f8"])
def test_explicit_edges_both_histogram_paths(cuda, kind, nb, wdt):
    """rows on every edge, below the first, on and above the last, NaN; nb <= 4096 bins use shared memory, more global"""
    from nbodykit_b200 import _lib
    smem = int(_lib.lib().nbk_zh_smem_bins())
    assert smem == 4096
    edges = _edges(kind, nb)
    rng = np.random.RandomState(nb)
    z = np.concatenate([rng.uniform(0.0, 1.1, 100000), edges, edges, [np.nan, -0.5, 1.5, np.nextafter(edges[0], 0)]])
    rng.shuffle(z)
    w = None if wdt is None else rng.uniform(size=z.size).astype(wdt)
    r = _check(z, w, edges)
    if w is None:
        assert (zo.counts(z, edges) >= 2).all()          # every edge holds two rows
    from nbodykit_b200.algorithms.zhist import _inverse_width
    assert (_inverse_width(edges) > 0) == (kind == "even")


@pytest.mark.parametrize("zdt", ["f4", "f8"])
def test_float32_rows_on_edges(cuda, zdt):
    """float32 redshifts equal to float64 edges compare exactly after widening"""
    e32 = np.linspace(0.1, 0.9, 41).astype("f4")
    edges = e32.astype("f8")
    z = np.concatenate([e32, e32, np.nextafter(e32, np.float32(0)), np.nextafter(e32, np.float32(2))]).astype(zdt)
    _check(z, None, edges)


def test_two_rows_and_one_row(cuda):
    r = _check(np.array([0.4, 0.6]))
    assert len(r.bin_edges) >= 2
    with pytest.raises(ValueError, match="zero spread"):
        _run(np.array([0.5]))
    with pytest.raises(ValueError, match="empty"):
        _run(np.zeros(0))
    with pytest.raises(ValueError, match="non-finite"):
        _run(np.array([0.5, np.nan, 0.7]))
    with pytest.raises(ValueError, match="non-finite"):
        _run(np.array([0.5, np.inf, 0.7]), bins=4)


def test_host_columns_and_rerun(cuda):
    z = zo.make_redshifts(9, 3000)
    a = _run(z, device=False)
    b = _run(z)
    np.testing.assert_array_equal(a.nbar, b.nbar)
    nbar = b.nbar.copy()
    b.run()
    np.testing.assert_array_equal(b.nbar, nbar)


def _reference_source(comm=None, weight=False):
    """the reference tests' catalogue: RandomCatalog(1000, seed=42) with z ~ N(0.5, 0.1) (and uniform weights)"""
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import RandomCatalog
    source = RandomCatalog(1000, seed=42, comm=comm or SelfComm())
    source['z'] = source.rng.normal(loc=0.5, scale=0.1)
    if weight:
        source['weight'] = source.rng.uniform(0, high=1.)
    return source


def test_reference_unweighted(cuda):
    from nbodykit_b200.lab import RedshiftHistogram
    r = RedshiftHistogram(_reference_source(), 1.0, _cosmo(), redshift='z')
    assert (r.nbar * r.dV).sum() == 1000


def test_reference_weighted(cuda):
    from nbodykit_b200.lab import RedshiftHistogram
    source = _reference_source(weight=True)
    r = RedshiftHistogram(source, 1.0, _cosmo(), redshift='z', weight='weight')
    np.testing.assert_allclose((r.nbar * r.dV).sum(), source['weight'].sum())


def test_reference_save(cuda, tmp_path):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import RedshiftHistogram
    r = RedshiftHistogram(_reference_source(), 1.0, _cosmo(), redshift='z')
    r.run()
    path = str(tmp_path / 'zhist-test.json')
    r.save(path)
    r2 = RedshiftHistogram.load(path, comm=SelfComm())
    np.testing.assert_array_equal(r.bin_edges, r2.bin_edges)
    np.testing.assert_array_equal(r.bin_centers, r2.bin_centers)
    np.testing.assert_array_equal(r.dV, r2.dV)
    np.testing.assert_array_equal(r.nbar, r2.nbar)
    for k in r.attrs:
        np.testing.assert_array_equal(r.attrs[k], r2.attrs[k])
    x = np.linspace(0.2, 0.8, 11)
    np.testing.assert_array_equal(r.interpolate(x), r2.interpolate(x))


@pytest.mark.parametrize("ext", ["extrapolate", "zeros", "const", 0, 1, 3])
@pytest.mark.parametrize("zdt", ["f4", "f8"])
def test_interpolate_matches_scipy(cuda, ext, zdt):
    z = zo.make_redshifts(84, 10000)
    r = _run(z)
    c, nbar = r.bin_centers, r.nbar
    t, _ = zo.spline(c, nbar)
    lo, hi = c[0], c[-1]
    x = np.concatenate([np.linspace(lo - 0.3, hi + 0.3, 20001), c, t, [lo, hi, np.nextafter(lo, 0), np.nextafter(hi, 2)],
                        z[:5000]]).astype(zdt)
    want = zo.interpolate(x, c, nbar, ext)
    tol = 1e-14 * np.abs(nbar).max()
    got = r.interpolate(x, ext)                                 # NumPy in, NumPy out
    assert isinstance(got, np.ndarray) and got.dtype == np.float64 and got.shape == x.shape
    np.testing.assert_allclose(got, want, rtol=0, atol=tol)
    dev = r.interpolate(torch.from_numpy(x).cuda(), ext)        # device in, device out
    assert isinstance(dev, torch.Tensor) and dev.is_cuda and dev.dtype == torch.float64
    np.testing.assert_array_equal(dev.cpu().numpy(), got)
    col = r.interpolate(_cat(x)["z"], ext)                      # a device Column
    assert isinstance(col, torch.Tensor) and col.is_cuda
    np.testing.assert_array_equal(col.cpu().numpy(), got)
    restated, _ = zo.splev(x, *zo.spline(c, nbar), ext)
    np.testing.assert_allclose(got, restated, rtol=0, atol=tol)


def test_interpolate_raise_and_shapes(cuda):
    z = zo.make_redshifts(84, 10000)
    r = _run(z)
    c = r.bin_centers
    inside = np.linspace(c[0], c[-1], 1001)
    np.testing.assert_allclose(r.interpolate(inside, 'raise'), zo.interpolate(inside, c, r.nbar, 'raise'), rtol=0,
                               atol=1e-14 * r.nbar.max())
    for bad in ([c[0] - 1e-9], [c[-1] + 0.1], [-0.5, 0.5]):
        with pytest.raises(ValueError, match="not in the domain"):
            r.interpolate(np.array(bad), 'raise')
        with pytest.raises(ValueError, match="not in the domain"):
            r.interpolate(torch.tensor(bad, device="cuda"), 2)
    s = r.interpolate(0.5)
    assert isinstance(s, np.ndarray) and s.shape == () and s == zo.interpolate(0.5, c, r.nbar)
    grid = r.interpolate(inside[:1000].reshape(10, 100))
    assert grid.shape == (10, 100)
    assert r.interpolate(np.zeros(0)).shape == (0,)
    nan = r.interpolate(np.array([np.nan, 0.5]))
    assert np.isnan(nan[0]) and np.isfinite(nan[1])
    # NZ as a catalogue column, scaled by alpha (the reference's test_with_zhist)
    cat = _cat(z)
    cat['NZ'] = r.interpolate(cat['z']) * 0.1
    np.testing.assert_allclose(cat['NZ'].compute().cpu().numpy(), zo.interpolate(z, c, r.nbar) * 0.1, rtol=0,
                               atol=1e-15 * r.nbar.max())


@pytest.mark.parametrize("name", ["scott", "explicit"])
def test_golden_fixtures(cuda, name):
    """the reference's own edges, nbar and interpolation, stored with their inputs"""
    g = np.load(os.path.join(GOLDEN, "zhist_%s.npz" % name))
    bins = None if name == "scott" else g["bin_edges"]
    r = _run(g["z"], None, bins)
    np.testing.assert_allclose(r.bin_edges, g["bin_edges"], rtol=1e-13, atol=0)
    np.testing.assert_allclose(r.nbar, g["nbar"], rtol=1e-13, atol=0)
    rw = _run(g["z"], g["w"], bins)
    np.testing.assert_allclose(rw.nbar, g["nbar_weighted"], rtol=1e-12, atol=0)
    tol = 1e-14 * np.abs(g["nbar"]).max() * 10
    for e in ("extrapolate", "zeros", "const"):
        np.testing.assert_allclose(r.interpolate(g["x"], e), g["interp_%s" % e], rtol=0, atol=tol)


def test_reference_save_file_loads_and_interpolates(cuda):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import RedshiftHistogram
    r = RedshiftHistogram.load(os.path.join(GOLDEN, "zhist_reference_save.json"), comm=SelfComm())
    g = np.load(os.path.join(GOLDEN, "zhist_scott.npz"))
    np.testing.assert_allclose(r.interpolate(g["x"], "zeros"), g["interp_zeros"], rtol=0, atol=1e-14 * g["nbar"].max())


def test_rows_beyond_2_31(cuda):
    """64-bit row indices: 2^31 + 5 float32 rows on one rank"""
    from nbodykit_b200.algorithms import zhist
    from nbodykit_b200.comm import SelfComm
    n = (1 << 31) + 5
    z = torch.full((n,), 0.25, dtype=torch.float32, device="cuda")
    z[-3:] = 0.75
    z[-1] = float("nan")
    m = zhist.local_moments(z)
    assert m[0] == n - 1 and m[5] == 1 and m[3] == 0.25 and m[4] == 0.75
    counts = zhist.histogram(z, None, np.array([0.0, 0.5, 1.0]), SelfComm())
    np.testing.assert_array_equal(counts, [n - 3, 2])
    del z
    torch.cuda.empty_cache()


def test_with_zhist_end_to_end(cuda):
    """the reference's test_conv_power.py::test_with_zhist through this package's ConvolvedFFTPower(Nmesh=128)"""
    from nbodykit_b200 import transform
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ConvolvedFFTPower, FKPCatalog, RandomCatalog, RedshiftHistogram
    cosmo = _cosmo()
    comm = SelfComm()
    data = RandomCatalog(zo.NDATA, seed=42, comm=comm)
    randoms = RandomCatalog(zo.NDATA * 10, seed=84, comm=comm)
    for s in [data, randoms]:
        s['z'] = s.rng.normal(loc=0.5, scale=0.1)
        s['ra'] = s.rng.uniform(low=110, high=260)
        s['dec'] = s.rng.uniform(low=-3.6, high=60.)
        s['Position'] = transform.SkyToCartesian(s['ra'], s['dec'], s['z'], cosmo=cosmo)
    zhist = RedshiftHistogram(randoms, zo.FSKY, cosmo, redshift='z')
    alpha = 1.0 * data.csize / randoms.csize
    randoms['NZ'] = zhist.interpolate(randoms['z']) * alpha
    data['NZ'] = zhist.interpolate(data['z']) * alpha
    fkp = FKPCatalog(data, randoms)
    r = ConvolvedFFTPower(fkp.to_mesh(Nmesh=128), poles=[0, 2, 4], dk=0.005)
    np.testing.assert_allclose(r.attrs['data.norm'], zo.DATA_NORM, rtol=1e-4)
    np.testing.assert_allclose(r.attrs['randoms.norm'], zo.RANDOMS_NORM, rtol=1e-4)
    data_norm, randoms_norm, nz_d, nz_r = zo.with_zhist_norms(cosmo)
    np.testing.assert_allclose(np.asarray(data['NZ']), nz_d, rtol=0, atol=1e-14 * nz_d.max())
    np.testing.assert_allclose(r.attrs['data.norm'], data_norm, rtol=1e-12)
    np.testing.assert_allclose(r.attrs['randoms.norm'], randoms_norm, rtol=1e-12)


# ---- several ranks over gloo, sharing device 0

def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, fn, args, ret):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
    try:
        from nbodykit_b200.comm import TorchComm
        ret[rank] = fn(TorchComm(), *args)
    finally:
        dist.destroy_process_group()


def _spawn(fn, world, *args):
    mgr = mp.Manager()
    try:
        ret = mgr.dict()
        mp.spawn(_worker, args=(world, _free_port(), fn, args, ret), nprocs=world, join=True)
        return [ret[r] for r in range(world)]
    finally:
        mgr.shutdown()


def _zh_ranks(comm, z, w, split, edges_list):
    mine = slice(split[comm.rank], split[comm.rank + 1])
    out = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for key, bins in [("scott", None), ("int", 9)] + [("edges%d" % k, e) for k, e in enumerate(edges_list)]:
            r = _run(z[mine], None if w is None else w[mine], bins, comm)
            out[key] = dict(edges=r.bin_edges, nbar=r.nbar, dV=r.dV)
        r = _run(z[mine], None, None, comm)
        x = np.linspace(0.0, 1.0, 101)
        out["interp"] = r.interpolate(x, "zeros")
        try:
            r.interpolate(np.array([5.0]) if comm.rank == comm.size - 1 else np.array([0.5]), "raise")
            out["raised"] = False
        except ValueError:
            out["raised"] = True
    return out


@pytest.mark.parametrize("P,empty,weighted", [(2, False, False), (2, True, True), (3, True, False), (3, False, True)])
def test_several_ranks(cuda, P, empty, weighted):
    z = zo.make_redshifts(17, 30000)
    w = np.random.RandomState(2).uniform(size=z.size) if weighted else None
    n = z.size
    split = list(np.linspace(0, n, P + 1).astype(int))
    if empty:
        split = [0, 0, n] if P == 2 else [0, n // 3, n // 3, n]
    edges_list = [_edges("nonuniform", 300), _edges("even", 5000)]
    res = _spawn(_zh_ranks, P, z, w, split, edges_list)
    for key in res[0]:
        if key in ("interp", "raised"):
            continue
        for r in res[1:]:          # bit-identical on every rank
            np.testing.assert_array_equal(r[key]["edges"], res[0][key]["edges"])
            np.testing.assert_array_equal(r[key]["nbar"], res[0][key]["nbar"])
        one = _run(z, w, None if key == "scott" else (9 if key == "int" else edges_list[int(key[5:])]))
        np.testing.assert_allclose(res[0][key]["edges"], one.bin_edges, rtol=1e-13, atol=0)
        assert len(res[0][key]["edges"]) == len(one.bin_edges)
        # counts on the same edges are equal; weighted sums within 1e-12 of sum |w|
        counts = zo.counts(z, res[0][key]["edges"], w)
        got = res[0][key]["nbar"] * res[0][key]["dV"]
        if w is None:
            np.testing.assert_array_equal(np.rint(got), counts)
            np.testing.assert_array_equal(res[0][key]["nbar"], counts / res[0][key]["dV"])
        else:
            assert (np.abs(got - counts) <= 1e-12 * zo.counts(z, res[0][key]["edges"], np.abs(w)) + 1e-300).all()
    assert all(r["raised"] for r in res)
    for r in res[1:]:
        np.testing.assert_array_equal(r["interp"], res[0]["interp"])
