"""FFT3PCF on the GPU: the two kernels against NumPy; the estimator against the float64 oracle (tests/fft3pcf_oracle.py)
in f8 and f4 on power-of-two, mixed-radix and Bluestein meshes; the exact link to SimulationBox3PCF on grid-node
objects; CatalogMesh inputs; invariance under the cube's axis transposes and reflections; the blocked path; P = 2, 3, 4
ranks sharing one GPU against one rank.  tests/mgpu_check_fft3pcf.py runs the several-GPU comparison under torchrun.

Tolerances: nsep is an integer count and must match exactly; |d corr_l| <= tol * bound_l with bound_l = (2l + 1) /
(16 pi^2) sum_x |delta| (sum_{s1} |delta|) (sum_{s2} |delta|), tol = 1e-10 (f8) or 1e-4 (f4)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import fft3pcf_oracle as fo
from test_gpu_bispectrum import SHAPES, TOL, _field, _mesh

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLES = [0, 1, 2, 3, 4]


def _edges(L, nb=5):
    """nb bins up to 0.45 of the smallest side"""
    return np.linspace(0, 0.45 * min(L), nb + 1)


def _run(mesh, poles=POLES, edges=None, **kw):
    from nbodykit_b200.lab import FFT3PCF
    return FFT3PCF(mesh, poles, edges, **kw)


def _corr(r, poles):
    return np.stack([r.poles["corr_%d" % ell] for ell in poles])


def _check(r, want, poles, tol, what):
    np.testing.assert_array_equal(r.nsep, want["nsep"], err_msg=what)
    got = _corr(r, poles)
    err = np.abs(got - want["corr"]) / want["bound"]
    assert err.max() <= tol, "%s: |d corr| / bound = %.3g > %g" % (what, err.max(), tol)
    ncells = np.prod(r.attrs["Nmesh"])
    nn = np.outer(r.nsep.astype("f8"), r.nsep.astype("f8"))
    for p, ell in enumerate(poles):
        np.testing.assert_allclose(r.poles["zeta_%d" % ell], 16 * np.pi ** 2 * got[p] / (ncells * nn), rtol=1e-14,
                                   err_msg=what)


# ---- the kernels
@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_kernel_fill_matches_real_ylm(cuda, dtype):
    """a run of m at one (l, b) on an x slab of a non-cubic odd mesh: the oracle's real Y_lm (scipy) on the bin"""
    from nbodykit_b200 import _lib
    from nbodykit_b200.algorithms.threeptcf import coefficient_table
    N, L = (22, 15, 18), (110., 90., 100.)
    e = np.array([3., 12.5, 26., 40.])
    x0, xn = 5, 9
    Lmax = 10
    T = _lib.darr(coefficient_table(Lmax).ravel())
    sx, sy, sz, r = fo.separations(N, L)
    b = fo.bins(N, L, e)
    tdt = torch.float64 if dtype == "f8" else torch.float32
    ncell = xn * N[1] * N[2]
    for ell, b_, m0, nm in ((0, 0, 0, 1), (3, 1, -3, 7), (10, 2, -10, 21), (7, 0, 2, 4), (10, 1, -4, 3)):
        out = torch.full((nm, ncell), 7.0, dtype=tdt, device="cuda")
        _lib.check(_lib.lib().nbk_fft3pcf_kernel_fill(out.data_ptr(), 8 if dtype == "f8" else 4, _lib.iarr(N),
                                                      _lib.darr(L), x0, xn, _lib.darr(e), len(e), b_, ell, m0, nm, T,
                                                      Lmax, ncell, None), "fill")
        got = out.cpu().numpy().astype("f8").reshape(nm, xn, N[1], N[2])
        for q in range(nm):
            want = np.where(b == b_, fo.real_ylm(ell, m0 + q, sx, sy, sz, r), 0.0)[x0:x0 + xn]
            atol = 1e-13 if dtype == "f8" else 3e-7
            np.testing.assert_allclose(got[q], want, rtol=0, atol=atol, err_msg="l=%d m=%d" % (ell, m0 + q))
            assert (got[q][b[x0:x0 + xn] != b_] == 0).all()


@pytest.mark.parametrize("dtype", ["f8", "f4"])
@pytest.mark.parametrize("na,nb", [(1, 1), (5, 5), (32, 32), (7, 3), (32, 29)])
def test_gram_matches_numpy(cuda, dtype, na, nb):
    """sum_x w a_i b_j, same set (i <= j only) and two sets, odd cell counts"""
    from nbodykit_b200 import _lib
    rng = np.random.RandomState(na * 100 + nb)
    ncell = 20001
    tdt = torch.float64 if dtype == "f8" else torch.float32
    code = 8 if dtype == "f8" else 4
    w = torch.from_numpy(rng.standard_normal(ncell)).to(tdt).cuda()
    A = torch.from_numpy(rng.standard_normal((na, ncell + 3))).to(tdt).cuda()     # padded rows: stride != ncell
    B = torch.from_numpy(rng.standard_normal((nb, ncell + 3))).to(tdt).cuda()
    wh, Ah, Bh = (t.cpu().numpy().astype("f8") for t in (w, A, B))
    bound = (np.abs(wh) * np.abs(Ah[:, :ncell])[:, None, :] * np.abs(Bh[:, :ncell])[None, :, :]).sum(-1)
    out = torch.full((na, nb), 1.5, dtype=torch.float64, device="cuda")       # accumulates
    _lib.check(_lib.lib().nbk_fft3pcf_gram(w.data_ptr(), A.data_ptr(), ncell + 3, na, B.data_ptr(), ncell + 3, nb, code,
                                           ncell, out.data_ptr(), None), "gram")
    want = 1.5 + (wh * Ah[:, None, :ncell] * Bh[None, :, :ncell]).sum(-1)
    assert (np.abs(out.cpu().numpy() - want) <= 1e-12 * bound).all()
    if na == nb:
        same = torch.zeros((na, na), dtype=torch.float64, device="cuda")
        _lib.check(_lib.lib().nbk_fft3pcf_gram(w.data_ptr(), A.data_ptr(), ncell + 3, na, A.data_ptr(), ncell + 3, na,
                                               code, ncell, same.data_ptr(), None), "gram")
        s = same.cpu().numpy()
        want = (wh * Ah[:, None, :ncell] * Ah[None, :, :ncell]).sum(-1)
        bound = (np.abs(wh) * np.abs(Ah[:, None, :ncell]) * np.abs(Ah[None, :, :ncell])).sum(-1)
        iu = np.triu_indices(na)
        assert (np.abs(s[iu] - want[iu]) <= 1e-12 * bound[iu]).all()
        assert (s[np.tril_indices(na, -1)] == 0).all()


# ---- the estimator
@pytest.mark.parametrize("dtype", ["f8", "f4"])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_matches_oracle(cuda, shape, dtype):
    N, L = SHAPES[shape]
    F = _field(N, 21)
    e = _edges(L)
    r = _run(_mesh(F, L, dtype), edges=e)
    Fm = F.astype(dtype).astype("f8")
    want = fo.fft_form(Fm, N, L, e, POLES)
    _check(r, want, POLES, TOL[dtype], "%s %s" % (shape, dtype))
    p = r.poles
    assert p.dims == ["r1", "r2"]
    assert p.data.dtype.names == tuple("corr_%d" % ell for ell in POLES) + tuple("zeta_%d" % ell for ell in POLES)
    for ell in POLES:
        np.testing.assert_array_equal(p["corr_%d" % ell], p["corr_%d" % ell].T)
    assert r.nsep.dtype == np.dtype("u8")
    from nbodykit_b200.algorithms.fft3pcf import bin_blocks, transform_count
    assert r.attrs["transforms"] == transform_count(bin_blocks(5, 5), POLES) == 1 + 2 * 5 * 25
    for key in ("poles", "edges", "Nmesh", "BoxSize", "transforms", "N1", "shotnoise"):
        assert key in r.attrs


@pytest.mark.parametrize("cplx,real", [("c16", "f8"), ("c8", "f4")])
def test_complex_mesh_equals_real(cuda, cplx, real):
    """a complex-typed mesh stores its real field as a real array: the same answer as the real-typed mesh"""
    N, L = SHAPES["48x36x30"]
    F = _field(N, 26)
    e = _edges(L)
    a = _run(_mesh(F, L, cplx), edges=e)
    b = _run(_mesh(F, L, real), edges=e)
    np.testing.assert_array_equal(a.nsep, b.nsep)
    bound = fo.bound(F, N, L, e, POLES)
    err = np.abs(_corr(a, POLES) - _corr(b, POLES)) / bound
    assert err.max() <= 1e-12, err.max()


def test_direct_form_16(cuda):
    """independent of every FFT and of Y_lm: the oracle's direct sum at 16 x 12 x 10"""
    N, L = (16, 12, 10), (160., 130., 90.)
    F = _field(N, 22)
    e = np.array([5., 17., 30., 44.])
    r = _run(_mesh(F, L, "f8"), edges=e)
    want = fo.direct_form(F, N, L, e, POLES)
    want["bound"] = fo.bound(F, N, L, e, POLES)
    _check(r, want, POLES, TOL["f8"], "direct")


def test_exact_link_to_simulationbox3pcf(cuda):
    """objects on grid nodes (H = 2), their count field F in a FieldMesh; SimulationBox3PCF on the objects plus one row
    of weight -mean(F) at every node is the same multilinear sum as FFT3PCF's corr_l, l = 0 .. 10.  The edges sit
    between the separations H sqrt(n)."""
    from nbodykit_b200.lab import ArrayCatalog, SimulationBox3PCF
    N, Lside = 32, 64.
    H = Lside / N
    L = (Lside,) * 3
    poles = list(range(11))
    e = H * np.sqrt(np.array([0.5, 4.5, 12.5, 30.5, 60.5, 100.5]))
    rng = np.random.RandomState(5)
    idx = rng.randint(0, N, size=(3000, 3))
    idx[:600] = idx[:600] % 4 + 10                                   # a clump: a strongly non-Gaussian field
    F = np.zeros((N,) * 3)
    np.add.at(F, tuple(idx.T), 1.0)
    mean = F.sum() / F.size
    r = _run(_mesh(F, L, "f8"), poles=poles, edges=e)
    nodes = np.indices((N,) * 3).reshape(3, -1).T
    pos = np.concatenate([idx, nodes]).astype("f8") * H
    w = np.concatenate([np.ones(len(idx)), np.full(len(nodes), -mean)])
    cat = ArrayCatalog({"Position": torch.from_numpy(pos).cuda(), "Weight": torch.from_numpy(w).cuda()}, BoxSize=L)
    ref = SimulationBox3PCF(cat, poles, e)
    bound = fo.bound(F, (N,) * 3, L, e, poles)
    got = _corr(r, poles)
    want = np.stack([ref.poles["corr_%d" % ell] for ell in poles])
    err = np.abs(got - want) / bound
    assert err.max() <= 1e-10, err.max()
    assert (np.abs(want[0]) / bound[0]).max() > 1e-3
    np.testing.assert_array_equal(r.nsep, fo.nsep((N,) * 3, L, e))


@pytest.mark.parametrize("resampler", ["nnb", "cic"])
def test_catalog_mesh(cuda, resampler):
    """a CatalogMesh gives the oracle's answer on its own to_real_field()"""
    from nbodykit_b200.lab import ArrayCatalog
    N, L = SHAPES["48x36x30"]
    rng = np.random.RandomState(8)
    pos = rng.uniform(0, 1, (20000, 3)) * np.asarray(L)
    pos[:4000] = pos[:4000] * 0.1 + np.asarray(L) * 0.3
    cat = ArrayCatalog({"Position": torch.from_numpy(pos).cuda()}, BoxSize=L)
    mesh = cat.to_mesh(Nmesh=N, BoxSize=L, resampler=resampler, compensated=False, dtype="f8")
    e = _edges(L)
    r = _run(mesh, edges=e)
    F = mesh.to_real_field().numpy()
    _check(r, fo.fft_form(F, N, L, e, POLES), POLES, TOL["f8"], resampler)
    assert r.attrs["N1"] == 20000


def test_transposes_and_reflections(cuda):
    """on a cube the statistic is invariant under the axis permutations and reflections of the grid (max(edges) < L/2:
    at |s_i| = L/2 the half-open wrap would not be reflected); every Y_lm, l = 0 .. 10, enters the sum over m"""
    N, L = (32, 32, 32), (200., 200., 200.)
    poles = list(range(11))
    F = _field(N, 23)
    F[3:9, 10:13, 20:30] += 4.0                                   # an anisotropic feature
    e = np.linspace(0, 90., 5)
    base = _corr(_run(_mesh(F, L, "f8"), poles=poles, edges=e), poles)
    bound = fo.bound(F, N, L, e, poles)
    variants = [np.transpose(F, (1, 0, 2)), np.transpose(F, (2, 1, 0)), np.transpose(F, (0, 2, 1)),
                np.transpose(F, (1, 2, 0))]
    variants += [np.roll(np.flip(F, a), 1, a) for a in range(3)]          # i -> -i (mod N)
    for k, G in enumerate(variants):
        got = _corr(_run(_mesh(np.ascontiguousarray(G), L, "f8"), poles=poles, edges=e), poles)
        err = np.abs(got - base) / bound
        assert err.max() <= 1e-10, (k, err.max())
    # not vacuous: the odd and high multipoles of this field are far from zero against the bound
    assert (np.abs(base[[1, 5, 10]]) / bound[[1, 5, 10]]).max() > 1e-6


@pytest.mark.parametrize("cap", [3, 4])
def test_blocked_path_matches_resident(cuda, monkeypatch, cap):
    from nbodykit_b200.algorithms.fft3pcf import bin_blocks, transform_count
    N, L = SHAPES["32"]
    F = _field(N, 24)
    e = _edges(L, 6)
    one = _run(_mesh(F, L, "f8"), edges=e)
    monkeypatch.setenv("NBK_BISPEC_RESIDENT", str(cap))
    blk = _run(_mesh(F, L, "f8"), edges=e)
    assert blk.attrs["transforms"] == transform_count(bin_blocks(6, cap), POLES) > one.attrs["transforms"]
    bound = fo.bound(F, N, L, e, POLES)
    err = np.abs(_corr(blk, POLES) - _corr(one, POLES)) / bound
    assert err.max() <= 1e-12, err.max()
    np.testing.assert_array_equal(blk.nsep, one.nsep)


def _on_ranks(comm, gid):
    from test_gpu_rank_statistics import GEOMS
    N, L, _, _ = GEOMS[gid]
    r = _run(_mesh(_field(N, 25), L, "f8", comm), edges=_edges(L))
    return dict(corr=_corr(r, POLES), nsep=r.nsep, transforms=r.attrs["transforms"])


@pytest.mark.parametrize("gid", ["32-P2", "32-P4", "48x36x30-P3", "44x22x26-P2"])
def test_ranks_match_one(cuda, gid):
    from test_gpu_rank_statistics import GEOMS
    from test_gpu_slab_route import _spawn
    N, L, P, _ = GEOMS[gid]
    F = _field(N, 25)
    e = _edges(L)
    one = _run(_mesh(F, L, "f8"), edges=e)
    bound = fo.bound(F, N, L, e, POLES)
    parts = _spawn(_on_ranks, P, gid)
    for rank, part in enumerate(parts):
        np.testing.assert_array_equal(part["nsep"], one.nsep)
        err = np.abs(part["corr"] - _corr(one, POLES)) / bound
        assert err.max() <= 1e-12, (gid, rank, err.max())
        assert part["transforms"] == one.attrs["transforms"]


def test_two_gpu_fft3pcf_matches_one_gpu():
    """launches tests/mgpu_check_fft3pcf.py under torchrun when the box has >= 2 GPUs"""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29549", os.path.join(ROOT, "tests", "mgpu_check_fft3pcf.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    sys.stdout.write(out.stdout[-3000:])
    sys.stderr.write(out.stderr[-3000:])
    assert out.returncode == 0
