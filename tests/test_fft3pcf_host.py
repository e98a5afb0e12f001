"""FFT3PCF without a GPU: the oracle's FFT form (scipy Y_lm, rfftn) equals its direct form (every pair of separations,
explicit Legendre polynomials); every argument error is raised before any paint or transform; the separation counts
against a direct count; the transform count and bin blocks; the table layout; save / load."""
import numpy as np
import pytest

import fft3pcf_oracle as fo

POLES = [0, 1, 2, 3, 4]


def _field(N, seed):
    rng = np.random.RandomState(seed)
    return rng.standard_normal(N) + 0.5 * rng.standard_normal(N) ** 2 + 2.0


@pytest.mark.parametrize("N,L,edges", [((12, 12, 12), (120., 120., 120.), [0., 14., 27., 41., 55.]),
                                       ((16, 12, 10), (160., 130., 90.), [5., 17., 30., 44.])])
def test_fft_form_equals_direct_form(N, L, edges):
    F = _field(N, 1)
    a = fo.fft_form(F, N, L, edges, POLES)
    b = fo.direct_form(F, N, L, edges, POLES)
    np.testing.assert_array_equal(a["nsep"], b["nsep"])
    assert (a["nsep"] > 0).all()
    err = np.abs(a["corr"] - b["corr"]) / a["bound"]
    assert err.max() <= 1e-12, err.max()
    # the statistic is far from zero against its bound: the comparison is not vacuous
    assert (np.abs(a["corr"][0]) / a["bound"][0]).max() > 1e-4
    np.testing.assert_allclose(a["zeta"], 16 * np.pi ** 2 * a["corr"] / (np.prod(N) * np.outer(a["nsep"], a["nsep"])),
                               rtol=1e-15)


class _Geometry:
    """a MeshSource of given geometry that fails if painted"""

    def __new__(cls, N=(16, 16, 16), L=(100., 100., 100.)):
        from nbodykit_b200.base.mesh import MeshSource

        class Geometry(MeshSource):
            def __init__(self):
                from nbodykit_b200.comm import SelfComm
                self.comm = SelfComm()
                self.attrs['Nmesh'] = np.array(N, dtype='i8')
                self.attrs['BoxSize'] = np.array(L, dtype='f8')

            def compute(self, *a, **k):
                raise AssertionError("painted")
        return Geometry()


@pytest.mark.parametrize("poles,edges", [
    ([], [0., 10.]), ([11], [0., 10.]), ([0, 0], [0., 10.]), ([2.5], [0., 10.]), ([-1], [0., 10.]), ([True], [0., 10.]),
    ([0], [10.]), ([0], [10., 5.]), ([0], [-1., 5.]), ([0], [0., np.inf]), ([0], np.linspace(0, 40, 34)),
    ([0], [0., 30., 50.1]),                  # max(edges) above half the smallest side (L = 100 x 120 x 140)
])
def test_bad_arguments_raise_before_device_work(monkeypatch, poles, edges):
    from nbodykit_b200.algorithms import fft3pcf
    monkeypatch.setattr(fft3pcf.FFT3PCF, "run", lambda self: pytest.fail("ran"))
    with pytest.raises(ValueError):
        fft3pcf.FFT3PCF(_Geometry(L=(100., 120., 140.)), poles, edges)


def test_good_arguments_reach_run(monkeypatch):
    """the same geometry with max(edges) = L/2 exactly passes the checks (and reaches run, which is stubbed)"""
    from nbodykit_b200.algorithms import fft3pcf
    ran = []
    monkeypatch.setattr(fft3pcf.FFT3PCF, "run", lambda self: ran.append(self.attrs))
    fft3pcf.FFT3PCF(_Geometry(L=(100., 120., 140.)), [0, 3, 10], [0., 25., 50.])
    assert ran and ran[0]['poles'] == [0, 3, 10]
    np.testing.assert_array_equal(ran[0]['edges'], [0., 25., 50.])
    with pytest.raises(TypeError):
        fft3pcf.FFT3PCF(object(), [0], [0., 10.])


@pytest.mark.parametrize("N,L,edges", [
    ((16, 16, 16), (64., 64., 64.), [0., 4., 4 * np.sqrt(2), 8., 12., 32.]),      # edges on separations: H = 4 exactly
    ((15, 9, 10), (150., 90., 100.), [0., 10., 20., 30., 45.]),                   # odd sides, edges on separations
    ((12, 20, 7), (100., 130., 77.), [1e-3, 7.3, 19.1, 38.5]),
])
def test_separation_counts_match_a_direct_count(N, L, edges):
    from nbodykit_b200.algorithms.fft3pcf import separation_counts
    got = separation_counts(N, L, edges)
    assert got.dtype == np.dtype('u8')
    # direct: every grid offset, its separation in (-N/2, N/2] cells, the contract's r and bin rule
    idx = np.indices(N).reshape(3, -1)
    n = [np.where(2 * idx[d] <= N[d], idx[d], idx[d] - N[d]) for d in range(3)]
    s = [n[d] * (L[d] / N[d]) for d in range(3)]
    r = np.sqrt((s[0] * s[0] + s[1] * s[1]) + s[2] * s[2])
    want = [int(((r > 0) & (r > edges[b]) & (r <= edges[b + 1])).sum()) for b in range(len(edges) - 1)]
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(got, fo.nsep(N, L, edges))


def test_transform_count_and_blocks():
    from nbodykit_b200.algorithms.fft3pcf import bin_blocks, transform_count
    assert bin_blocks(8, 8) == [list(range(8))] and bin_blocks(8, 64) == [list(range(8))]
    assert bin_blocks(8, 5) == [[0, 1], [2, 3], [4, 5], [6, 7]]
    assert bin_blocks(7, 6) == [[0, 1, 2], [3, 4, 5], [6]]
    poles = list(range(11))
    assert transform_count(bin_blocks(8, 8), poles) == 1 + 2 * 8 * 121
    # blocks of 2: block p is built 1 + p times per (l, m)
    assert transform_count(bin_blocks(8, 5), [0, 2]) == 1 + 2 * 6 * (2 + 4 + 6 + 8)


def _table():
    from nbodykit_b200.algorithms.fft3pcf import pole_table
    corr = np.arange(2 * 9, dtype='f8').reshape(2, 3, 3) + 1
    corr = corr + corr.transpose(0, 2, 1)
    nsep = np.array([4, 0, 6], dtype='u8')
    return corr, nsep, pole_table(corr, nsep, 64, [3, 0])


def test_pole_table_layout():
    corr, nsep, d = _table()
    assert d.dtype.names == ('corr_3', 'corr_0', 'zeta_3', 'zeta_0')
    np.testing.assert_array_equal(d['corr_3'], corr[0])
    np.testing.assert_array_equal(d['corr_0'], corr[1])
    assert d['zeta_0'][0, 2] == 16 * np.pi ** 2 * corr[1, 0, 2] / (64 * 4 * 6)
    assert np.isnan(d['zeta_3'][1]).all() and np.isnan(d['zeta_3'][:, 1]).all()


def test_save_load_round_trip(tmp_path):
    from nbodykit_b200.algorithms.fft3pcf import FFT3PCF
    from nbodykit_b200.binned_statistic import BinnedStatistic
    from nbodykit_b200.comm import SelfComm
    corr, nsep, d = _table()
    e = np.array([0., 10., 20., 30.])
    r = object.__new__(FFT3PCF)
    r.comm = SelfComm()
    r.attrs = dict(poles=[3, 0], edges=e, Nmesh=np.array([4, 4, 4]), BoxSize=np.array([60.] * 3), transforms=43,
                   N1=100, shotnoise=0.)
    r.nsep = nsep
    r.poles = BinnedStatistic(['r1', 'r2'], [e, e], d)
    path = str(tmp_path / "fft3pcf.json")
    r.save(path)
    s = FFT3PCF.load(path, comm=SelfComm())
    assert s.poles.dims == ['r1', 'r2']
    np.testing.assert_array_equal(s.poles.edges['r1'], e)
    for f in d.dtype.names:
        np.testing.assert_array_equal(s.poles[f], r.poles[f])
    assert s.nsep.dtype == np.dtype('u8')
    np.testing.assert_array_equal(s.nsep, nsep)
    assert s.attrs['poles'] == [3, 0] and s.attrs['transforms'] == 43
    np.testing.assert_array_equal(s.attrs['Nmesh'], [4, 4, 4])
