"""The three-point function without a GPU: the CPU restatement in oracle/threeptcf_oracle.py against the reference's
golden C++ result and against an O(N^2) Legendre brute force, the coefficient table against scipy's spherical
harmonics, argument validation of SimulationBox3PCF and of nbk_threeptcf, and save / load."""
import math

import numpy as np
import pytest

from oracle import threeptcf_oracle as to  # noqa: E402

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


def _close(got, want, tol):
    """|got - want| <= tol * B entrywise"""
    err = np.abs(got["zeta"] - want["zeta"])
    assert (err <= tol * want["bound"]).all(), float(np.max(err / np.maximum(want["bound"], 1e-300)))


def test_oracle_reproduces_golden_cpp_result():
    """1000 weighted points in L = 400, 8 bins over [0, 200], l = 0 .. 10: the file prints 7 significant digits"""
    pos, w, truth = to.golden()
    r = to.compute(pos, np.linspace(0, 200., 9), list(range(11)), box=[400.] * 3, w=w)
    for ell in range(11):
        np.testing.assert_allclose(r["zeta"][ell] * (4 * np.pi) ** 2 / (2 * ell + 1), truth[..., ell], rtol=1e-6,
                                   err_msg="l = %d" % ell)
    assert (np.abs(r["zeta"]) <= r["bound"] * (1 + 1e-12)).all()


@pytest.mark.parametrize("case", range(4))
def test_oracle_matches_brute_force(case):
    rng = np.random.RandomState(50 + case)
    L = 20.
    n = 300
    pos = rng.uniform(size=(n, 3)) * L
    pos[:10] = pos[10:20]                                     # duplicates: r = 0 never counts
    box, edges = [L] * 3, np.linspace(0., 6., 5)
    w = rng.uniform(-1., 2., n) if case % 2 else None
    if case == 1:
        pos = (pos - 3.).astype("f4")                         # rows below 0 and f4 wrapping
    if case == 2:
        box = None                                            # not periodic
        edges = np.linspace(1., 7., 4)
    if case == 3:
        box = [L, 14., 17.]                                   # a non-cubic periodic box
        pos = np.mod(pos, box)
    poles = [0, 1, 2, 5, 10] if case != 3 else [3]
    a = to.compute(pos, edges, poles, box=box, w=w)
    b = to.brute_force(pos, edges, poles, box=box, w=w)
    np.testing.assert_array_equal(a["npairs"], b["npairs"])
    np.testing.assert_allclose(a["bound"], b["bound"], rtol=1e-13)
    _close(a, b, 1e-12)
    assert a["npairs"].sum() > 1000


def test_oracle_lattice_edges_left_open_right_closed():
    g = np.arange(6, dtype="f8")
    pos = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    r = to.compute(pos, [1., 2., 3.], [0], box=[6.] * 3)
    # r = 1 is on e_0 and excluded; (1, 2]: r^2 = 2, 3, 4 (12 + 8 + 6); (2, 3]: r^2 = 5, 6, 8, 9 (24 + 24 + 12 + 27,
    # with only +3 of the offsets +-3 in the minimum image d in (-3, 3])
    assert list(r["npairs"]) == [216 * 26, 216 * 87]


def test_coefficient_table_against_sph_harm_y():
    from scipy.special import sph_harm_y
    from nbodykit_b200.algorithms.threeptcf import coefficient_table, max_ell
    L = max_ell()
    assert L >= 10
    T = coefficient_table(L)
    rng = np.random.RandomState(3)
    u = rng.normal(size=(200, 3))
    u /= np.linalg.norm(u, axis=1)[:, None]
    theta, phi = np.arccos(u[:, 2]), np.arctan2(u[:, 1], u[:, 0])
    xy = u[:, 0] + 1j * u[:, 1]
    zk = u[:, 2][:, None] ** np.arange(L + 1)
    for ell in range(L + 1):
        for m in range(ell + 1):
            off = m * (L + 1) - m * (m - 1) // 2
            y = xy ** m * (zk @ T[off + ell - m]) / math.sqrt(4 * math.pi)
            np.testing.assert_allclose(y, sph_harm_y(ell, m, theta, phi), rtol=0, atol=1e-12 * math.sqrt(2 * ell + 1),
                                       err_msg="l = %d, m = %d" % (ell, m))
            # Q_lm has the parity of l - m
            assert (T[off + ell - m][(ell - m + 1) % 2::2] == 0).all() and (T[off + ell - m][ell - m + 1:] == 0).all()


@pytest.fixture
def no_run(monkeypatch):
    from nbodykit_b200.algorithms.threeptcf import SimulationBox3PCF
    monkeypatch.setattr(SimulationBox3PCF, "run", lambda self, pedantic=False: None)


def test_validation(no_run):
    from nbodykit_b200.algorithms.threeptcf import max_bins, max_ell
    from nbodykit_b200.lab import SimulationBox3PCF as T
    cat = _cat()
    e = np.linspace(0., 10., 5)
    r = T(cat, [1, 0], e)
    assert r.attrs["poles"] == [1, 0] and r.attrs["periodic"] and r.attrs["weight"] == "Weight"
    assert set(r.attrs) == {"poles", "edges", "BoxSize", "periodic", "weight", "position"}
    with pytest.raises(ValueError, match="missing"):
        T(cat, [0], e, weight="nope")
    with pytest.raises(ValueError, match="BoxSize must be supplied"):
        T(_cat(BoxSize=None), [0], e)
    with pytest.raises(ValueError, match="Rmax > BoxSize/2"):
        T(cat, [0], np.linspace(0., 50.1, 4))
    with pytest.raises(ValueError, match="Rmax > BoxSize/2"):
        T(_cat(BoxSize=[100., 100., 50.]), [0], [1., 30.])
    T(cat, [0], np.linspace(0., 50.1, 4), periodic=False)
    T(_cat(BoxSize=[100., 80., 60.]), [0], [1., 30.]) # non-cubic periodic boxes are fine
    for bad in ([2., 1.], [1.], [-1., 2.], [0., np.inf], [[1., 2.]]):
        with pytest.raises(ValueError, match="edges"):
            T(cat, [0], bad)
    for bad in ([], [0, 0], [-1], [1.5], "ab", [True]):
        with pytest.raises(ValueError, match="poles"):
            T(cat, bad, e)
    with pytest.raises(ValueError, match="l = %d" % max_ell()):
        T(cat, [max_ell() + 1], e)
    with pytest.raises(ValueError, match="at most %d" % max_bins()):
        T(cat, [0], np.linspace(0., 10., max_bins() + 2))
    T(cat, list(range(max_ell() + 1)), np.linspace(0., 10., max_bins() + 1))


def test_kernel_entry_validates_before_cuda():
    from nbodykit_b200 import _lib
    from nbodykit_b200.algorithms.threeptcf import coefficient_table
    L = _lib.lib()
    box, nc, tol = _lib.darr([10.] * 3), _lib.iarr([4] * 3), _lib.darr([0.] * 3)
    err = lambda: L.nbk_last_error()  # noqa: E731
    T = _lib.darr(coefficient_table(10).ravel())

    def call(edges=(1., 2.), poles=(0,), nch=1, nc_=nc, coef=T):
        return L.nbk_threeptcf(None, None, None, None, nch, None, None, None, None, 1, 1, box, nc_, tol, _lib.darr(edges),
                               len(edges), _lib.i32arr(poles), len(poles), coef, None, None, None, None, None)
    assert call(edges=(1.,)) == -1 and b"edges" in err()
    assert call(edges=tuple(range(35))) == -1 and b"radial bins" in err()
    assert call(edges=(2., 1.)) == -1 and b"increase" in err()
    assert call(edges=(-1., 1.)) == -1 and b"non-negative" in err()
    assert call(poles=()) == -1 and b"poles" in err()
    assert call(poles=(11,)) == -1 and b"pole 11" in err()
    assert call(poles=(2, 2)) == -1 and b"twice" in err()
    assert call(coef=None) == -1 and b"coefficient" in err()
    assert call(nc_=_lib.iarr([4, 0, 4])) == -1 and b"cell count" in err()
    assert call(nch=-1) == -1 and b"chunk count" in err()
    assert call(nch=0, poles=tuple(range(11)), edges=tuple(range(33))) == 0          # nothing to count, at the caps
    assert L.nbk_threeptcf_max_ell() == 10 and L.nbk_threeptcf_max_bins() == 32
    assert L.nbk_threeptcf_chunk_rows() >= 32


def test_save_load_round_trip(tmp_path):
    from nbodykit_b200.binned_statistic import BinnedStatistic
    from nbodykit_b200.lab import SimulationBox3PCF
    edges = np.linspace(0., 10., 4)
    data = np.zeros((3, 3), dtype=[("corr_1", "f8"), ("corr_0", "f8")])
    data["corr_0"] = np.arange(9.).reshape(3, 3) / 7.
    data["corr_1"] = -np.arange(9.).reshape(3, 3) * np.pi
    r = object.__new__(SimulationBox3PCF)
    r.poles = BinnedStatistic(["r1", "r2"], [edges, edges], data)
    r.attrs = dict(poles=[1, 0], edges=edges, BoxSize=np.array([10.] * 3), periodic=True, weight="w", position="Position")
    r.comm = _cat().comm
    f = str(tmp_path / "t.json")
    r.save(f)
    s = SimulationBox3PCF.load(f, comm=r.comm)
    np.testing.assert_array_equal(s.poles.data, r.poles.data)
    assert s.poles.dims == ["r1", "r2"] and s.poles.variables == ["corr_1", "corr_0"]
    np.testing.assert_array_equal(s.poles.edges["r1"], edges)
    assert s.attrs["poles"] == [1, 0] and s.attrs["weight"] == "w"


def test_class_is_exported():
    import nbodykit_b200.algorithms as A
    import nbodykit_b200.lab as lab
    assert lab.SimulationBox3PCF is A.SimulationBox3PCF
    assert "SimulationBox3PCF" in A.__all__
