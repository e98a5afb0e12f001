"""Pair counts without a GPU: argument validation of SimulationBoxPairCount / SimulationBox2PCF and of nbk_paircount,
the analytic randoms, the estimators, wp, to_poles, save / load, and the CPU restatement in oracle/paircount_oracle.py
against an O(N^2) brute force."""
import numpy as np
import pytest

from oracle import paircount_oracle as po  # noqa: E402


_COMM = []


def _cat(n=20, box=100., seed=0, **attrs):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ArrayCatalog
    if not _COMM:
        _COMM.append(SelfComm())
    pos = np.random.RandomState(seed).uniform(size=(n, 3)) * box
    kw = dict(BoxSize=attrs.pop("BoxSize", [box] * 3))
    if kw["BoxSize"] is None:
        kw = {}
    kw.update(attrs)
    return ArrayCatalog({"Position": pos, "Weight": np.ones(n)}, comm=_COMM[0], **kw)


@pytest.fixture
def no_run(monkeypatch):
    from nbodykit_b200.algorithms.paircount import SimulationBoxPairCount
    monkeypatch.setattr(SimulationBoxPairCount, "run", lambda self: None)


def test_pair_count_validation(no_run):
    from nbodykit_b200.lab import SimulationBoxPairCount as PC
    cat = _cat()
    e = np.linspace(1, 10, 5)
    with pytest.raises(ValueError, match="allowed 'mode'"):
        PC("3d", cat, e)
    with pytest.raises(ValueError, match="greater than zero"):
        PC("1d", cat, [0., 1., 2.])
    with pytest.raises(ValueError, match="'Nmu' keyword is required"):
        PC("2d", cat, e)
    with pytest.raises(ValueError, match="mode should be '2d'"):
        PC("1d", cat, e, Nmu=5)
    with pytest.raises(ValueError, match="'pimax' keyword is required"):
        PC("projected", cat, e)
    with pytest.raises(ValueError, match="mode should be 'projected'"):
        PC("1d", cat, e, pimax=10.)
    with pytest.raises(ValueError, match="at least 1.0"):
        PC("projected", cat, e, pimax=0.5)
    with pytest.raises(ValueError, match="``los`` should be one of"):
        PC("1d", cat, e, los="w")
    with pytest.raises(ValueError, match=r"\[0,1,2\]"):
        PC("1d", cat, e, los=5)
    with pytest.raises(ValueError, match="'Weight2' is missing"):
        from nbodykit_b200.comm import SelfComm
        from nbodykit_b200.lab import ArrayCatalog
        PC("1d", ArrayCatalog({"Position": np.zeros((3, 3))}, comm=SelfComm(), BoxSize=10.), e, weight="Weight2")
    with pytest.raises(ValueError, match="'Pos' is missing"):
        PC("1d", cat, e, position="Pos")
    with pytest.raises(ValueError, match="cross-correlation sources"):
        PC("1d", cat, e, second=_cat(BoxSize=[50.] * 3))
    with pytest.raises(ValueError, match="sources and the pair count algorithm"):
        PC("1d", cat, e, BoxSize=50.)
    with pytest.raises(ValueError, match="BoxSize must be supplied"):
        PC("1d", _cat(BoxSize=None), e)
    with pytest.raises(ValueError, match="Rmax > BoxSize/2"):
        PC("1d", cat, [1., 60.])
    with pytest.raises(ValueError, match="Rmax > BoxSize/2"):
        PC("projected", cat, e, pimax=51.)
    with pytest.raises(NotImplementedError, match="non-cubic"):
        PC("1d", _cat(BoxSize=[100., 100., 80.]), e)
    # the package's own checks
    for bad in ([[1., 2.], [3., 4.]], [1., np.inf], [1., 3., 2.], [1., 1., 2.], [5.]):
        with pytest.raises(ValueError, match="edges must be"):
            PC("1d", cat, bad)
    with pytest.raises(NotImplementedError, match="RA/Dec"):
        PC("angular", cat, e)
    # non-periodic boxes need not be cubic; config and show_progress are recorded
    r = PC("1d", _cat(BoxSize=[100., 100., 80.]), e, periodic=False, show_progress=True, nthreads=4)
    assert r.attrs["config"] == {"nthreads": 4} and r.attrs["show_progress"] is True
    r = PC("projected", cat, e, pimax=20., los="x")
    assert r.attrs["los"] == 0 and r.attrs["N1"] == 20 and r.attrs["N2"] is None
    assert PC("1d", cat, e, los=-1).attrs["los"] == 2
    for k in ("mode", "edges", "Nmu", "pimax", "N1", "N2", "BoxSize", "periodic", "weight", "position", "config", "los"):
        assert k in r.attrs


def test_2pcf_needs_randoms_when_not_periodic(no_run):
    from nbodykit_b200.lab import SimulationBox2PCF
    with pytest.raises(ValueError, match="randoms1"):
        SimulationBox2PCF("1d", _cat(), [1., 5.], periodic=False)


def test_row_limit():
    from nbodykit_b200.algorithms.paircount import _check_rows
    _check_rows((1 << 31) - 1, "x")
    with pytest.raises(ValueError, match="2\\^31 - 1"):
        _check_rows(1 << 31, "x")


def test_kernel_entry_validates_before_cuda():
    from nbodykit_b200 import _lib
    L = _lib.lib()
    box, nc, tol = _lib.darr([10.] * 3), _lib.iarr([4] * 3), _lib.darr([0.] * 3)
    err = lambda: L.nbk_last_error()  # noqa: E731

    def call(mode=1, edges=(1., 2.), e2=None, pimax=0.0, nc_=nc, nch=1):
        ea = _lib.darr(edges)
        e2a = _lib.darr(e2) if e2 is not None else None
        return L.nbk_paircount(mode, None, None, None, None, nch, None, None, None, None, 1, 1, box, nc_, tol, ea, len(edges),
                               e2a, len(e2) if e2 is not None else 0, pimax, None, None, None, None, None, None)
    assert call(mode=7) == -1 and b"bad mode" in err()
    assert call(edges=(1.,)) == -1 and b"edges" in err()
    assert call(edges=(2., 1.)) == -1 and b"increase" in err()
    assert call(edges=(0., 1.)) == -1 and b"positive" in err()
    assert call(mode=2) == -1 and b"second-dimension" in err()
    assert call(mode=3, e2=(0., 1.), pimax=float("nan")) == -1 and b"pimax" in err()
    assert call(nc_=_lib.iarr([4, 0, 4])) == -1 and b"cell count" in err()
    assert call(nch=-1) == -1 and b"chunk count" in err()
    assert call(nch=0) == 0                                       # nothing to count
    assert L.nbk_paircount_chunk_rows() >= 32 and L.nbk_paircount_smem_bins() >= 64
    keys = _lib.iarr([0])
    assert L.nbk_fof_grid_keys(None, 3, 1, 1, box, None, nc, keys, None) == -1 and b"dtype" in err()
    assert L.nbk_fof_grid_keys(None, 4, 1, 1, None, None, nc, keys, None) == -1 and b"required" in err()
    assert L.nbk_fof_grid_keys(None, 4, 0, 1, box, None, nc, keys, None) == 0


def test_filling_factors_closed_forms():
    from nbodykit_b200.algorithms.paircount import filling_factor
    V = 1000. ** 3
    r = np.array([1., 2., 5.])
    np.testing.assert_allclose(filling_factor("1d", {"r": r}, [1000.] * 3),
                               [4 / 3. * np.pi * (8 - 1) / V, 4 / 3. * np.pi * (125 - 8) / V], rtol=1e-14)
    mu = np.linspace(0, 1, 5)
    f = filling_factor("2d", {"r": r, "mu": mu}, [1000.] * 3)
    assert f.shape == (2, 4)
    # a full shell splits evenly over |mu|
    np.testing.assert_allclose(f[0], 4 / 3. * np.pi * 7 / V / 4, rtol=1e-14)
    np.testing.assert_allclose(f.sum(1), filling_factor("1d", {"r": r}, [1000.] * 3), rtol=1e-14)
    pi = np.linspace(0, 40, 41)
    f = filling_factor("projected", {"rp": r, "pi": pi}, [1000.] * 3)
    # annulus area times 2 dpi (both signs of pi)
    np.testing.assert_allclose(f[1, 3], np.pi * (25 - 4) * 2 * 1. / V, rtol=1e-14)


def _pairs(mode, dims, edges, wn, n=None, total=1., **attrs):
    from nbodykit_b200.lab import BinnedStatistic
    shape = tuple(len(e) - 1 for e in edges)
    data = np.zeros(shape, dtype=[(dims[0], "f8"), ("npairs", "u8"), ("wnpairs", "f8")])
    data["wnpairs"] = wn
    data["npairs"] = wn if n is None else n
    data[dims[0]] = np.arange(np.prod(shape)).reshape(shape) + 0.5
    pc = type("PC", (), {})()
    pc.pairs = BinnedStatistic(dims, edges, data, fields_to_sum=["npairs", "wnpairs"])
    pc.attrs = dict(mode=mode, total_wnpairs=total, **attrs)
    return pc


def test_natural_estimator_on_hand_built_counts():
    from nbodykit_b200.algorithms.paircount import filling_factor, natural_estimator
    r = np.array([1., 2., 3.])
    N, L = 100, 10.
    ff = filling_factor("1d", {"r": r}, [L] * 3)
    DD = _pairs("1d", ["r"], [r], np.array([2.0, 1.5]) * N * N * ff, total=0.5 * N * (N - 1), N1=N, N2=None, is_cross=False,
                BoxSize=np.array([L] * 3))
    RR, corr = natural_estimator(DD)
    np.testing.assert_allclose(RR["wnpairs"], N * N * ff, rtol=1e-14)
    np.testing.assert_allclose(corr["corr"], [1.0, 0.5], rtol=1e-12)
    np.testing.assert_array_equal(corr["r"], DD.pairs["r"])
    # cross: N1 N2 normalisation
    DD = _pairs("1d", ["r"], [r], N * 2 * N * ff, total=0.5 * N * 2 * N, N1=N, N2=2 * N, is_cross=True, BoxSize=np.array([L] * 3))
    np.testing.assert_allclose(natural_estimator(DD)[1]["corr"], 0., atol=1e-12)


def test_landy_szalay_wp_and_poles_on_hand_built_counts():
    from nbodykit_b200.algorithms.paircount import landy_szalay, projected_wp, WedgeBinnedStatistic
    rp, pi = np.array([1., 2., 4.]), np.linspace(0, 3, 4)
    shape = (2, 3)
    DD = _pairs("projected", ["rp", "pi"], [rp, pi], np.full(shape, 8.), total=4.)
    DR = _pairs("projected", ["rp", "pi"], [rp, pi], np.full(shape, 6.), total=6.)
    RD = _pairs("projected", ["rp", "pi"], [rp, pi], np.full(shape, 3.), total=3.)
    rrw = np.full(shape, 2.)
    rrn = np.ones(shape, "u8")
    rrn[1, 2] = 0
    RR = _pairs("projected", ["rp", "pi"], [rp, pi], rrw, n=rrn, total=2.)
    with pytest.warns(UserWarning, match="NaN"):
        corr = landy_szalay(DD, DR, RD, RR)
    # (2/4 * 8 - 2/6 * 6 - 2/3 * 3) / 2 + 1 = 1
    want = np.ones(shape)
    want[1, 2] = np.nan
    np.testing.assert_allclose(corr["corr"], want)
    assert isinstance(corr, WedgeBinnedStatistic)
    corr["corr"] = np.array([[1., 2., 3.], [0.5, 0.5, 0.5]])
    wp = projected_wp(corr)
    assert wp.dims == ["rp"]
    np.testing.assert_allclose(wp["corr"], [2 * 6., 2 * 1.5])
    # to_poles of wedges constant in mu: monopole = the value, quadrupole = the discretised Legendre average
    mu = np.linspace(0, 1, 5)
    w = _pairs("2d", ["r", "mu"], [rp, mu], np.ones((2, 4)), total=1.).pairs
    data = np.zeros((2, 4), dtype=[("corr", "f8"), ("r", "f8")])
    data["corr"] = np.array([[3.] * 4, [1., 2., 3., 4.]])
    data["r"] = [[1.5] * 4, [3.] * 4]
    xi = WedgeBinnedStatistic(["r", "mu"], [rp, mu], data)
    poles = xi.to_poles([0, 2])
    np.testing.assert_allclose(poles["corr_0"], [3., 2.5])
    c = 0.5 * (mu[1:] + mu[:-1])
    np.testing.assert_allclose(poles["corr_2"][1], (5 * 0.5 * (3 * c ** 2 - 1) * np.array([1., 2, 3, 4]) * 0.25).sum())
    np.testing.assert_allclose(poles["r"], [1.5, 3.])
    assert poles.attrs["poles"] == [0, 2] and w.shape == (2, 4)


def test_save_load_round_trip(tmp_path):
    from nbodykit_b200.algorithms.paircount import (SimulationBox2PCF, SimulationBoxPairCount, WedgeBinnedStatistic,
                                                    natural_estimator, projected_wp)
    from nbodykit_b200.comm import SelfComm
    rp, pi = np.array([1., 2., 4.]), np.linspace(0, 3, 4)
    pc = object.__new__(SimulationBoxPairCount)
    src = _pairs("projected", ["rp", "pi"], [rp, pi], np.arange(6.).reshape(2, 3) + 1, total=7.)
    pc.pairs, pc.comm = src.pairs, SelfComm()
    pc.attrs = dict(mode="projected", edges=rp, Nmu=None, pimax=3., N1=10, N2=None, BoxSize=np.array([10.] * 3), periodic=True,
                    weight="Weight", position="Position", config={}, los=2, total_wnpairs=7., is_cross=False, show_progress=False)
    pc.save(str(tmp_path / "pc.json"))
    back = SimulationBoxPairCount.load(str(tmp_path / "pc.json"), comm=SelfComm())
    assert back.pairs.dims == ["rp", "pi"] and back.pairs.data.dtype == pc.pairs.data.dtype
    np.testing.assert_array_equal(back.pairs.data, pc.pairs.data)
    np.testing.assert_array_equal(back.pairs.edges["pi"], pi)
    assert back.attrs["total_wnpairs"] == 7. and back.attrs["los"] == 2

    t = object.__new__(SimulationBox2PCF)
    t.comm = SelfComm()
    t.attrs = dict(pc.attrs)
    RR, t.corr = natural_estimator(pc)
    t.D1D2, t.R1R2, t.D1R2, t.D2R1 = pc.pairs.copy(cls=WedgeBinnedStatistic), RR, None, None
    t.wp = projected_wp(t.corr)
    t.save(str(tmp_path / "tpcf.json"))
    u = SimulationBox2PCF.load(str(tmp_path / "tpcf.json"), comm=SelfComm())
    np.testing.assert_array_equal(u.corr["corr"], t.corr["corr"])
    np.testing.assert_array_equal(u.wp["corr"], t.wp["corr"])
    np.testing.assert_array_equal(u.D1D2["npairs"], t.D1D2["npairs"])
    assert u.D1R2 is None and isinstance(u.R1R2, WedgeBinnedStatistic) and u.wp.dims == ["rp"]


def test_classes_are_exported():
    import nbodykit_b200.algorithms as alg
    import nbodykit_b200.lab as lab
    for name in ("SimulationBoxPairCount", "SimulationBox2PCF"):
        assert name in alg.__all__ and getattr(lab, name) is getattr(alg, name)


@pytest.mark.parametrize("mode", ["1d", "2d", "projected"])
@pytest.mark.parametrize("periodic", [True, False])
def test_oracle_matches_brute_force(mode, periodic):
    rng = np.random.RandomState(3)
    L = 50.
    a = po.clustered(1, L, 400, 3, 30, 1.5, dtype="f4")
    b = (rng.uniform(size=(300, 3)) * L).astype("f8")
    w1, w2 = rng.uniform(0.5, 2, len(a)), rng.uniform(0.5, 2, len(b))
    box = [L] * 3 if periodic else None
    edges = np.linspace(0.5, 12., 7)
    kw = dict(Nmu=7 if mode == "2d" else None, pimax=9.5 if mode == "projected" else None)
    for los in (2, 0):
        for args in (dict(), dict(pos2=b, w2=w2)):
            got = po.count(a, mode, edges, box, w1=w1, los=los, **args, **kw)
            want = po.brute_force(a, mode, edges, box, w1=w1, los=los, **args, **kw)
            np.testing.assert_array_equal(got["npairs"], want["npairs"])
            np.testing.assert_allclose(got["wnpairs"], want["wnpairs"], rtol=1e-12)
            np.testing.assert_allclose(got["sepsum"], want["sepsum"], rtol=1e-12)
            assert got["npairs"].sum() > 100


def test_oracle_lattice_edges():
    """pairs exactly on bin edges fall in the upper bin; pairs at s = 0 never count"""
    g = np.arange(4.)
    pos = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    out = po.count(pos, "1d", [1., 2., 3.], [4.] * 3)
    # periodic 4^3 lattice: separations 1 (6 neighbours), sqrt2 (12), sqrt3 (8) in [1, 2); 2 (6 at distance 2 along an
    # axis, which wraps onto itself: 3 distinct... each of the 3 axes once) lands in [2, 3)
    assert out["npairs"][0] == 64 * (6 + 12 + 8)
    brute = po.brute_force(pos, "1d", [1., 2., 3.], [4.] * 3)
    np.testing.assert_array_equal(out["npairs"], brute["npairs"])
