"""Survey pair counts (SurveyDataPairCount, SurveyData2PCF) and SurveyData3PCF on the GPU against the CPU restatement in
oracle/survey_paircount_oracle.py: npairs exactly equal, the double sums to rtol 1e-12.  Covers every mode, auto and
cross, weighted and not, f4 and f8 sky columns, a uniform survey patch and a clustered lognormal shell, pairs along one
line of sight, through the observer and on chord edges, angular edges up to 90 degrees, permuted input, survey '1d'
against the non-periodic box count, the Landy-Szalay estimator, the reference's survey 3PCF test, and P = 2 and 3
processes over gloo sharing device 0; tests/mgpu_check_survey.py runs the same comparison under torchrun."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import survey_paircount_oracle as so  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_COMM = []
_LOGNORMAL = []


def _comm():
    from nbodykit_b200.comm import SelfComm
    if not _COMM:
        _COMM.append(SelfComm())
    return _COMM[0]


def _cat(ra, dec, z=None, w=None, comm=None, dtype="f8"):
    from nbodykit_b200.lab import ArrayCatalog
    data = {"RA": torch.as_tensor(np.ascontiguousarray(ra, dtype)).cuda(),
            "DEC": torch.as_tensor(np.ascontiguousarray(dec, dtype)).cuda()}
    if z is not None:
        data["Redshift"] = torch.as_tensor(np.ascontiguousarray(z, dtype)).cuda()
    if w is not None:
        data["Weight"] = torch.as_tensor(np.ascontiguousarray(w)).cuda()
    return ArrayCatalog(data, comm=comm or _comm())


def _rows(mode, ra, dec, z, dtype="f8"):
    """the float64 rows the algorithm counts: SkyToCartesian (SkyToUnitSphere for 'angular') of the columns as
    stored"""
    from nbodykit_b200 import transform as T
    from nbodykit_b200.cosmology import Planck15
    t = [torch.as_tensor(np.ascontiguousarray(a, dtype)).cuda() for a in (ra, dec, z)]
    p = T.SkyToUnitSphere(t[0], t[1]) if mode == "angular" else T.SkyToCartesian(t[0], t[1], t[2], Planck15)
    return p.cpu().numpy()


def _compare(r, want):
    p = r.pairs
    np.testing.assert_array_equal(p["npairs"], want["npairs"])
    assert p["npairs"].dtype == np.uint64
    np.testing.assert_allclose(p["wnpairs"], want["wnpairs"], rtol=1e-12, atol=0)
    n = want["npairs"]
    sep = np.where(n > 0, want["sepsum"] / np.maximum(n, 1), 0.)
    np.testing.assert_allclose(p[p.dims[0]], sep, rtol=1e-12, atol=0)


def _kw(mode, Nmu=8, pimax=40.):
    return dict(Nmu=Nmu if mode == "2d" else None, pimax=pimax if mode == "projected" else None)


def _run(mode, s1, edges, s2=None, w1=None, w2=None, dtype="f8", **kw):
    """s1, s2: (ra, dec, z) arrays"""
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200.lab import SurveyDataPairCount
    first = _cat(*s1, w=w1, dtype=dtype)
    second = _cat(*s2, w=w2, dtype=dtype) if s2 is not None else None
    r = SurveyDataPairCount(mode, first, edges, cosmo=Planck15, second=second, **kw)
    want = so.count(_rows(mode, *s1, dtype=dtype), mode, edges,
                    pos2=None if s2 is None else _rows(mode, *s2, dtype=dtype), w1=w1, w2=w2, **kw)
    _compare(r, want)
    assert r.attrs["is_cross"] == (s2 is not None)
    assert r.candidates >= int(want["npairs"].sum())
    return r, want


def _lognormal():
    """(ra, dec, z) of a clustered shell 100 < r < 280 Mpc/h cut from a LogNormalCatalog, observer at the box centre"""
    if not _LOGNORMAL:
        from nbodykit_b200 import transform as T
        from nbodykit_b200.cosmology import NoWiggleEHPower, Planck15
        from nbodykit_b200.lab import LogNormalCatalog
        cat = LogNormalCatalog(Plin=NoWiggleEHPower(), nbar=2e-4, BoxSize=600., Nmesh=64, bias=2.0, seed=21,
                               comm=_comm())
        pos = cat["Position"].compute().double() - 300.
        r = torch.linalg.vector_norm(pos, dim=1)
        pos = pos[(r > 100.) & (r < 280.)]
        ra, dec, z = T.CartesianToSky(pos, Planck15)
        _LOGNORMAL.append(tuple(a.cpu().numpy() for a in (ra, dec, z)))
    return _LOGNORMAL[0]


# ---- catalogues against the oracle -----------------------------------------------------------------------------------
_CASES = [  # dtype, cross, weights, catalogue
    ("f8", False, False, "uniform"),
    ("f4", True, True, "uniform"),
    ("f4", False, True, "lognormal"),
    ("f8", True, False, "lognormal"),
]
_EDGES = {  # (uniform, lognormal)
    "1d": (np.linspace(10, 150, 10), np.linspace(2., 40., 8)),
    "2d": (np.linspace(10, 150, 10), np.linspace(2., 40., 8)),
    "projected": (np.linspace(10, 150, 10), np.linspace(2., 30., 8)),
    "angular": (np.array([0.5, 2., 10., 30., 60., 90.]), np.logspace(-1, 1, 6)),
}


@pytest.mark.parametrize("mode", ["1d", "2d", "projected", "angular"])
@pytest.mark.parametrize("case", range(len(_CASES)))
def test_against_oracle(cuda, mode, case):
    dtype, cross, weighted, kind = _CASES[case]
    rng = np.random.RandomState(200 + case)
    if kind == "uniform":
        s1 = so.sky_catalogue(case, 1500 if mode == "angular" else 6000)
        s2 = so.sky_catalogue(case + 50, 1000 if mode == "angular" else 4000) if cross else None
        edges = _EDGES[mode][0]
    else:
        full = _lognormal()
        n = len(full[0])
        i1 = rng.permutation(n)[:n // 2] if cross else np.arange(n)
        s1 = tuple(a[i1] for a in full)
        s2 = tuple(a[rng.permutation(n)[:n // 3]] for a in full) if cross else None
        edges = _EDGES[mode][1]
    w1 = rng.uniform(0.5, 2., len(s1[0])) if weighted else None
    w2 = rng.uniform(0.5, 2., len(s2[0])) if (weighted and cross) else None
    r, want = _run(mode, s1, edges, s2, w1, w2, dtype=dtype, **_kw(mode, pimax=80. if kind == "uniform" else 30.))
    assert want["npairs"].sum() > 20000
    if mode == "2d":
        assert (want["npairs"].sum(0) > 0).all()          # every mu bin is populated


# ---- constructed pairs -----------------------------------------------------------------------------------------------
def test_constructed_pairs(cuda):
    """pairs along one line of sight (mu = 1), through the observer (l = 0) and on chord edges"""
    from nbodykit_b200.algorithms.paircount import count_pairs
    rng = np.random.RandomState(7)
    ra, dec, z = so.sky_catalogue(9, 400, ra=(20., 40.), dec=(10., 25.), z=(0.05, 0.005))
    zk = np.linspace(0.03, 0.06, 10)
    theta = np.array([0.5, 1., 2., 4.])
    ra = np.concatenate([ra, ra[:50], np.repeat([0., 180.], 10), np.repeat([0.] + list(theta), 4)])
    dec = np.concatenate([dec, dec[:50], np.zeros(20), np.zeros(20)])
    zz = np.concatenate([z, z[:50] * 1.02, zk, zk, np.full(20, 0.05)])
    s = (ra, dec, zz)
    r, want = _run("2d", s, np.linspace(1., 300., 7), Nmu=10)
    assert want["npairs"][:, -1].sum() >= 100                # mu = 1: the 50 radial pairs, both orders
    r, want = _run("projected", s, np.linspace(1., 300., 7), pimax=300.)
    assert want["npairs"][:, 0].sum() >= 20                  # pi ~ 0: the pairs through the observer
    r, want = _run("angular", s, theta)                      # rows theta edges apart on the equator
    assert want["npairs"].sum() > 0
    _run("1d", s, np.linspace(1., 300., 7), w1=rng.uniform(size=len(ra)))
    # exact l = 0 (x2 = -x1) and exact mu = 1 (x2 = 2 x1) on rows given directly to the count
    x = _rows("1d", *s)[:200]
    rows = np.concatenate([x, -x[:50], 2. * x[50:100]])
    t = torch.from_numpy(rows).cuda()
    w = torch.ones(len(rows), dtype=torch.float64, device="cuda")
    e = np.linspace(1., 500., 6)
    for mode, kw in (("2d", dict(Nmu=7)), ("projected", dict(pimax=400.))):
        n, ws, ss, _ = count_pairs(mode, t, w, t, w, e, False, None, Nmu=kw.get("Nmu"), pimax=kw.get("pimax"),
                                   survey=True)
        want = so.count(rows, mode, e, **kw)
        np.testing.assert_array_equal(n.cpu().numpy().reshape(want["npairs"].shape), want["npairs"])
        np.testing.assert_allclose(ss.cpu().numpy().reshape(want["npairs"].shape), want["sepsum"], rtol=1e-12)
        assert want["npairs"][:, 0].sum() >= 100                # l = 0: mu = 0 and pi = 0
        if mode == "2d":
            assert want["npairs"][:, -1].sum() >= 100


def test_angular_wide_edges_all_sky(cuda):
    """theta up to 90 degrees over the whole sky: one or two cells per axis"""
    rng = np.random.RandomState(8)
    n = 1500
    ra = rng.uniform(0., 360., n)
    dec = np.rad2deg(np.arcsin(rng.uniform(-1., 1., n)))
    for edges in ([1., 30., 60., 90.], [45., 90.], [100., 150., 180.]):
        r, want = _run("angular", (ra, dec, np.ones(n)), np.asarray(edges))
        assert want["npairs"].sum() > 1000
    # mean theta of uniform points on the sphere in [0, 180): about 90 degrees
    r, _ = _run("angular", (ra, dec, np.ones(n)), np.array([1e-3, 180.]))
    assert abs(r.pairs["theta"][0] - 90.) < 2.


def test_permuted_input_same_counts(cuda):
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200.lab import SurveyDataPairCount
    s = _lognormal()
    w = np.random.RandomState(9).uniform(size=len(s[0]))
    p = np.random.RandomState(10).permutation(len(s[0]))
    edges = np.linspace(2., 30., 6)
    for mode, kw in (("2d", dict(Nmu=5)), ("projected", dict(pimax=20.)), ("angular", {})):
        e = np.logspace(-1, 1, 5) if mode == "angular" else edges
        r1 = SurveyDataPairCount(mode, _cat(*s, w=w), e, cosmo=Planck15, **kw)
        r2 = SurveyDataPairCount(mode, _cat(*(a[p] for a in s), w=w[p]), e, cosmo=Planck15, **kw)
        np.testing.assert_array_equal(r1.pairs["npairs"], r2.pairs["npairs"])
        np.testing.assert_allclose(r1.pairs["wnpairs"], r2.pairs["wnpairs"], rtol=1e-12)


class _ExactCosmo(object):
    """a cosmology that only takes NumPy arrays: Planck15's own distances, computed on the host"""

    def comoving_distance(self, z):
        from nbodykit_b200.cosmology import Planck15
        z = np.asarray(z, dtype="f8")                    # raises on a device tensor
        return Planck15.comoving_distance(z)


class _TableCosmo(object):
    """a NumPy-only cosmology without efunc: numpy.interp over a table of Planck15 distances"""

    def __init__(self):
        from nbodykit_b200.cosmology import Planck15
        self.z = np.linspace(0., 3., 30001)
        self.d = Planck15.comoving_distance(self.z)

    def comoving_distance(self, z):
        return np.interp(np.asarray(z, dtype="f8"), self.z, self.d)


def test_numpy_only_cosmology(cuda):
    """any object with comoving_distance(z) works: it is called on host arrays"""
    from nbodykit_b200 import transform as T
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200.lab import SurveyDataPairCount
    s = _lognormal()
    t = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in s]
    edges = np.linspace(2., 30., 6)
    for cosmo in (_ExactCosmo(), _TableCosmo()):
        rows = T.SkyToCartesian(t[0], t[1], t[2], cosmo)
        assert rows.is_cuda
        # Planck15's own distances to rounding; the table's to its interpolation error (dz^2 / 8 |chi''| < 1e-5)
        tol = 1e-12 if isinstance(cosmo, _ExactCosmo) else 1e-5
        np.testing.assert_allclose(rows.cpu().numpy(), _rows("1d", *s), rtol=0, atol=tol)
        for mode, kw in (("2d", dict(Nmu=5)), ("projected", dict(pimax=20.))):
            r = SurveyDataPairCount(mode, _cat(*s), edges, cosmo=cosmo, **kw)
            _compare(r, so.count(rows.cpu().numpy(), mode, edges, **kw))
            p = SurveyDataPairCount(mode, _cat(*s), edges, cosmo=Planck15, **kw)
            if isinstance(cosmo, _ExactCosmo):
                np.testing.assert_array_equal(r.pairs["npairs"], p.pairs["npairs"])
            else:                                        # within the table's interpolation error
                d = np.abs(r.pairs["npairs"].astype("i8") - p.pairs["npairs"].astype("i8")).sum()
                assert d <= 1e-4 * p.pairs["npairs"].sum()
        # the inverse on device tensors: Newton steps with the grid's slope when there is no efunc
        ra, dec, z = T.CartesianToSky(rows, cosmo)
        assert z.is_cuda
        np.testing.assert_allclose(T.SkyToCartesian(ra, dec, z, cosmo).cpu().numpy(), rows.cpu().numpy(), rtol=0,
                                   atol=1e-9)


def _bad_redshift(comm, bad_rank):
    """every rank holds a few rows; rank `bad_rank` has one redshift of -1.  Returns whether this rank raised"""
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200.lab import SurveyDataPairCount
    ra, dec, z = so.sky_catalogue(60 + comm.rank, 200)
    if comm.rank == bad_rank:
        z[7] = -1.
    try:
        SurveyDataPairCount("1d", _cat(ra, dec, z, comm=comm), np.linspace(5., 50., 4), cosmo=Planck15)
    except ValueError as e:
        return "above -1" in str(e)
    return False


def test_redshift_at_or_below_minus_one_raises_on_every_rank(cuda):
    from test_gpu_fof import _spawn
    assert _bad_redshift(_comm(), 0)
    assert _spawn(_bad_redshift, 2, 1) == [True, True]


def test_survey_1d_equals_box_count(cuda):
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200.lab import ArrayCatalog, SimulationBoxPairCount, SurveyDataPairCount
    s = _lognormal()
    edges = np.linspace(2., 40., 8)
    r = SurveyDataPairCount("1d", _cat(*s), edges, cosmo=Planck15)
    pos = torch.from_numpy(_rows("1d", *s)).cuda()
    box = SimulationBoxPairCount("1d", ArrayCatalog({"Position": pos}, comm=_comm(), BoxSize=[600.] * 3), edges,
                                 periodic=False)
    np.testing.assert_array_equal(r.pairs["npairs"], box.pairs["npairs"])
    np.testing.assert_allclose(r.pairs["r"], box.pairs["r"], rtol=1e-12)
    assert r.pairs["npairs"].sum() > 10000


def test_save_load(cuda, tmp_path):
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200.lab import SurveyDataPairCount
    s = so.sky_catalogue(11, 2000)
    for mode, kw in (("projected", dict(pimax=40.)), ("angular", {})):
        r = SurveyDataPairCount(mode, _cat(*s), np.linspace(10., 100., 5) if mode != "angular" else [1., 5., 20.],
                                cosmo=Planck15, **kw)
        f = str(tmp_path / ("pc_%s.json" % mode))
        r.save(f)
        q = SurveyDataPairCount.load(f, comm=_comm())
        assert q.attrs["cosmo"] == Planck15 and q.pairs.dims == r.pairs.dims
        np.testing.assert_array_equal(q.pairs["npairs"], r.pairs["npairs"])
        np.testing.assert_array_equal(q.pairs["wnpairs"], r.pairs["wnpairs"])


# ---- correlation functions -------------------------------------------------------------------------------------------
def test_landy_szalay_against_oracle_counts(cuda, tmp_path):
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200.lab import SurveyData2PCF, SurveyDataPairCount
    d = _lognormal()
    rng = np.random.RandomState(12)
    nr = 2 * len(d[0])
    # randoms: the data's redshifts, isotropic directions over the whole sky
    rr = (rng.uniform(0., 360., nr), np.rad2deg(np.arcsin(rng.uniform(-1., 1., nr))), rng.choice(d[2], nr))
    nd = len(d[0])
    for mode, edges, kw in (("1d", np.linspace(2., 30., 6), {}), ("2d", np.linspace(2., 30., 6), dict(Nmu=4)),
                            ("projected", np.linspace(2., 30., 6), dict(pimax=20.)),
                            ("angular", np.logspace(-0.5, 0.7, 5), {})):
        t = SurveyData2PCF(mode, _cat(*d), _cat(*rr), edges, cosmo=Planck15, **kw)
        pd, pr = _rows(mode, *d), _rows(mode, *rr)
        DD, DR, RR = (so.count(pd, mode, edges, **kw), so.count(pd, mode, edges, pos2=pr, **kw),
                      so.count(pr, mode, edges, **kw))
        fDD = (0.5 * (nr * nr - nr)) / (0.5 * (nd * nd - nd))
        fDR = (0.5 * (nr * nr - nr)) / (0.5 * nd * nr)
        want = (fDD * DD["wnpairs"] - 2 * fDR * DR["wnpairs"]) / RR["wnpairs"] + 1
        np.testing.assert_array_equal(t.D1D2["npairs"], DD["npairs"])
        np.testing.assert_array_equal(t.D1R2["npairs"], DR["npairs"])
        np.testing.assert_array_equal(t.R1R2["npairs"], RR["npairs"])
        np.testing.assert_allclose(t.corr["corr"], want, rtol=1e-12)
        if mode == "projected":
            np.testing.assert_allclose(t.wp["corr"], 2 * (want * np.diff(t.corr.edges["pi"])).sum(-1), rtol=1e-12)
            RRpc = SurveyDataPairCount(mode, _cat(*rr), edges, cosmo=Planck15, **kw)
            u = SurveyData2PCF(mode, _cat(*d), _cat(*rr), edges, cosmo=Planck15, R1R2=RRpc, **kw)
            np.testing.assert_array_equal(u.corr["corr"], t.corr["corr"])
            assert u.R1R2 is not None
            f = str(tmp_path / "tpcf.json")
            u.save(f)
            v = SurveyData2PCF.load(f, comm=_comm())
            np.testing.assert_array_equal(v.wp["corr"], u.wp["corr"])
            assert v.attrs["cosmo"] == Planck15
        else:
            assert t.wp is None
    # a cross correlation: randoms2 defaults to randoms1
    d2 = tuple(a[::2] for a in d)
    t = SurveyData2PCF("1d", _cat(*d), _cat(*rr), np.linspace(2., 30., 6), cosmo=Planck15, data2=_cat(*d2))
    assert t.randoms2 is t.randoms1
    pd2 = _rows("1d", *d2)
    np.testing.assert_array_equal(t.D1D2["npairs"], so.count(_rows("1d", *d), "1d", np.linspace(2., 30., 6),
                                                             pos2=pd2)["npairs"])


def test_survey_3pcf_reference_test(cuda, tmp_path):
    """the reference's test_survey_threeptcf: SurveyData3PCF equals SimulationBox3PCF(periodic=False) on the same rows"""
    from oracle import threeptcf_oracle as to
    from nbodykit_b200 import transform as T
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200.lab import ArrayCatalog, SimulationBox3PCF, SurveyData3PCF
    pos, w, _ = to.golden()
    pos = torch.from_numpy(pos - 200.).cuda()
    ra, dec, z = T.CartesianToSky(pos, Planck15)
    rows = T.SkyToCartesian(ra, dec, z, Planck15)
    cat = ArrayCatalog({"Position": rows, "RA": ra, "DEC": dec, "Z": z, "w": torch.from_numpy(w).cuda()},
                       comm=_comm())
    edges = np.linspace(0, 200.0, 9)
    ells = list(range(0, 11))
    ref = SimulationBox3PCF(cat, ells, edges, BoxSize=400., weight='w', periodic=False)
    r = SurveyData3PCF(cat, ells, edges, Planck15, weight='w', ra='RA', dec='DEC', redshift='Z')
    bound = to.compute(rows.cpu().numpy(), edges, ells, box=None, w=w)["bound"]
    for i, ell in enumerate(ells):
        err = np.abs(r.poles['corr_%d' % ell] - ref.poles['corr_%d' % ell])
        assert (err <= 1e-12 * bound[i]).all(), ell
    np.testing.assert_array_equal(r.npairs, ref.npairs)
    f = str(tmp_path / "3pcf.json")
    r.save(f)
    q = SurveyData3PCF.load(f, comm=_comm())
    assert q.attrs["cosmo"] == Planck15
    np.testing.assert_array_equal(q.poles["corr_2"], r.poles["corr_2"])


# ---- several ranks over gloo on device 0 -----------------------------------------------------------------------------
def _ranks(comm, mode, s1, s2, w1, edges, kw, split1, split2, dtype):
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200.lab import SurveyDataPairCount

    def cat(s, w, split):
        mine = slice(split[comm.rank], split[comm.rank + 1])
        return _cat(*(a[mine] for a in s), w=None if w is None else w[mine], comm=comm, dtype=dtype)
    first = cat(s1, w1, split1)
    second = cat(s2, None, split2) if s2 is not None else None
    r = SurveyDataPairCount(mode, first, edges, cosmo=Planck15, second=second, **kw)
    return dict(npairs=r.pairs["npairs"], wnpairs=r.pairs["wnpairs"], sep=r.pairs[r.pairs.dims[0]])


_MULTI = [  # P, mode, cross, empty rank
    (2, "2d", False, False),
    (3, "projected", True, True),
    (3, "angular", False, False),
    (2, "1d", True, True),
]


@pytest.mark.parametrize("case", range(len(_MULTI)))
def test_several_ranks_equal_one(cuda, case):
    from test_gpu_fof import _spawn
    P, mode, cross, empty = _MULTI[case]
    full = _lognormal()
    n = len(full[0])
    s1 = full
    s1 = tuple(a[np.argsort(full[0], kind="stable")] for a in full) if case % 2 else s1     # sorted by RA, or not
    s2 = tuple(a[np.random.RandomState(case).permutation(n)[:n // 2]] for a in full) if cross else None
    w1 = np.random.RandomState(case).uniform(0.5, 2., n)
    edges = np.logspace(-1, 1, 6) if mode == "angular" else np.linspace(2., 30., 7)
    kw = _kw(mode, pimax=20.)
    dtype = "f4" if case % 2 else "f8"

    def split(m):
        if empty:
            return [0, 0] + [m * (r + 1) // (P - 1) for r in range(P - 1)]
        return [r * m // P for r in range(P + 1)]
    parts = _spawn(_ranks, P, mode, s1, s2, w1, edges, kw, split(n), split(len(s2[0])) if cross else None, dtype)
    one = so.count(_rows(mode, *s1, dtype=dtype), mode, edges,
                   pos2=None if s2 is None else _rows(mode, *s2, dtype=dtype), w1=w1, **kw)
    for p in parts:
        np.testing.assert_array_equal(p["npairs"], one["npairs"])
        np.testing.assert_allclose(p["wnpairs"], one["wnpairs"], rtol=1e-12)
        np.testing.assert_array_equal(p["npairs"], parts[0]["npairs"])
    assert one["npairs"].sum() > 10000


def test_two_gpu_survey_matches_one_gpu():
    """launches tests/mgpu_check_survey.py under torchrun when the box has >= 2 GPUs"""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29535", os.path.join(ROOT, "tests", "mgpu_check_survey.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    sys.stdout.write(out.stdout[-3000:])
    sys.stderr.write(out.stderr[-3000:])
    assert out.returncode == 0
