"""FFTBispectrum multipoles without a GPU: the float64 oracle's FFT form against its FFT-free direct sum, the weighted
rows (pole_triples), the (b, c)-symmetric table with NaN off the evaluated triples, argument validation before any
device work, and save/load with and without multipoles."""
import json

import numpy as np
import pytest

import bispectrum_poles_oracle as bpo
from nbodykit_b200.algorithms import bispectrum as bs
from nbodykit_b200.comm import SelfComm
from oracle import bispectrum_oracle as bo

LOS = {"z": [0, 0, 1], "x": [1, 0, 0], "diag": list(np.ones(3) / np.sqrt(3))}


@pytest.mark.parametrize("los", sorted(LOS))
@pytest.mark.parametrize("N,L", [((12, 12, 12), (100., 100., 100.)), ((15, 15, 15), (80., 80., 80.)),
                                 ((16, 12, 10), (100., 70., 60.))], ids=["12", "15-odd", "16x12x10"])
def test_oracle_fft_form_equals_direct_sum(N, L, los):
    rng = np.random.RandomState(7)
    half = np.fft.rfftn(rng.normal(size=N) + 0.3 * rng.normal(size=N) ** 2) / np.prod(N)
    dk = 2 * np.pi / min(L)
    kedges = np.arange(0., np.pi * min(N) / max(L) + dk / 2, dk)
    a = bpo.fft_form_poles(half, N, L, kedges, [0, 2, 4], LOS[los])
    b = bpo.direct_form_poles(half, N, L, kedges, [0, 2, 4], LOS[los])
    for ell in (0, 2, 4):
        np.testing.assert_array_equal(a[ell]["triangles"], b[ell]["triangles"])
        ok = a[ell]["triangles"] > 0
        assert ok.sum() > 5
        np.testing.assert_array_equal(np.isnan(a[ell]["B"]), ~ok)
        assert (np.abs(a[ell]["B"] - b[ell]["B"])[ok] <= 1e-12 * a[ell]["bound"][ok]).all(), ell
    # ell = 0 is the plain estimator
    plain = bo.fft_form(half, N, L, kedges)
    index = {tuple(t): q for q, t in enumerate(plain["triples"].tolist())}
    q = [index[tuple(sorted(r))] for r in a[0]["rows"].tolist()]
    ok = a[0]["triangles"] > 0
    np.testing.assert_allclose(a[0]["B"][ok], plain["B"][q][ok], rtol=1e-12)


def test_oracle_mu_is_float32_arithmetic():
    """mu from float32 coordinates in the (kx l0 + ky l1) + kz l2 order, and L_ell by the recurrence"""
    mu = bpo.mu_half((8, 8, 8), (50., 50., 50.), LOS["diag"])
    assert mu.dtype == np.float32 and mu[0, 0, 0] == 0
    assert np.abs(mu).max() <= 1 + 1e-6
    x = np.linspace(-1, 1, 11)
    np.testing.assert_allclose(bpo.legendre(2, x), 1.5 * x ** 2 - 0.5, atol=1e-15)
    np.testing.assert_allclose(bpo.legendre(4, x), (35 * x ** 4 - 30 * x ** 2 + 3) / 8, atol=1e-15)


@pytest.mark.parametrize("kedges", [np.arange(0., 6.), np.arange(0.5, 6.5), np.array([0., 0.1, 0.2, 0.3])])
def test_pole_triples_coverage(kedges):
    tri = bs.shell_triples(kedges)
    rows = bs.pole_triples(kedges)
    assert rows.dtype == np.int32 and rows.shape[1] == 3
    assert (rows[:, 1] <= rows[:, 2]).all()
    assert len({tuple(r) for r in rows.tolist()}) == len(rows)
    # every row's sorted form is evaluated; each triple has one row per distinct weighted position
    sorted_rows = [tuple(sorted(r)) for r in rows.tolist()]
    evaluated = {tuple(t) for t in tri.tolist()}
    assert set(sorted_rows) == evaluated
    for t in evaluated:
        assert sorted_rows.count(t) == len(set(t)), t
    n_scalene = sum(len(set(t)) == 3 for t in evaluated)
    n_iso = sum(len(set(t)) == 2 for t in evaluated)
    n_equi = sum(len(set(t)) == 1 for t in evaluated)
    assert n_scalene > 0 and n_iso > 0 and n_equi > 0
    assert len(rows) == 3 * n_scalene + 2 * n_iso + n_equi
    np.testing.assert_array_equal(rows, bpo.pole_rows(kedges))


def test_poles_table_symmetric_and_nan():
    e = np.array([0., 0.1, 0.2, 0.3])
    tri = bs.shell_triples(e)
    rows = bs.pole_triples(e)
    rng = np.random.RandomState(4)
    N3 = 1000.
    counts = rng.randint(1, 5, size=len(tri))
    counts[1] = 0
    Tsum = counts * N3
    d = bs.bispectrum_table(e, [0.15, 0.25, 0.35], tri, rng.normal(size=len(tri)), Tsum, 8.0, N3)
    W = {2: rng.normal(size=len(rows)), 4: rng.normal(size=len(rows))}
    p = bs.poles_table(d, tri, rows, W, Tsum, 8.0, [0, 2, 4])
    assert p.shape == (3, 3, 3)
    assert p.dtype.names == ('k1', 'k2', 'k3', 'B_0', 'B_2', 'B_4', 'triangles')
    np.testing.assert_array_equal(p['B_0'], d['B'])
    np.testing.assert_array_equal(p['triangles'], d['triangles'])
    index = {tuple(t): q for q, t in enumerate(tri.tolist())}
    for ell in (2, 4):
        B = p['B_%d' % ell]
        np.testing.assert_array_equal(B, np.transpose(B, (0, 2, 1)))          # symmetric in (b, c)
        for r, w in zip(rows.tolist(), W[ell]):
            q = index[tuple(sorted(r))]
            if counts[q]:
                assert B[tuple(r)] == (2 * ell + 1) * 64.0 * w / Tsum[q]
            else:
                assert np.isnan(B[tuple(r)])
        # NaN exactly where the sorted triple holds no evaluated triangle
        np.testing.assert_array_equal(np.isnan(B), d['triangles'] == 0)
    assert p['triangles'][0, 0, 2] == 0 and np.isnan(p['B_2'][0, 0, 2]) and np.isnan(p['B_2'][2, 0, 0])
    # weights sit on k1: B_2 is not symmetric under exchanging k1 and k2
    i, j, l = next(t for t in tri.tolist() if len(set(t)) == 3 and counts[index[tuple(t)]])
    assert p['B_2'][i, j, l] != p['B_2'][j, i, l]


@pytest.mark.parametrize("poles,match", [([1], "odd multipole"), ([0, 2, 3], "imaginary"), ([10], "0 <= ell <= 8"),
                                         ([-2], "0 <= ell <= 8"), ([2.5], "even integers"), ([2, 2], "repeated")])
def test_bad_poles_raise_before_device_work(poles, match):
    # `first` is not even a mesh: the check runs before anything touches it
    with pytest.raises(ValueError, match=match):
        bs.FFTBispectrum(None, poles=poles)


@pytest.mark.parametrize("los,match", [([0, 0, 2], "unit vector"), ([1, 1, 0], "unit vector"), ([0, 1], "length 3"),
                                       (1.0, "length 3")])
def test_bad_los_raises_before_device_work(los, match):
    with pytest.raises(ValueError, match=match):
        bs.FFTBispectrum(None, poles=[2], los=los)


def test_check_poles_accepts():
    assert bs.check_poles(None, [0, 0, 1]) == []
    assert bs.check_poles([0, 2, 4, 6, 8], [1, 0, 0]) == [0, 2, 4, 6, 8]
    assert bs.check_poles(np.array([4, 2]), list(np.ones(3) / np.sqrt(3))) == [4, 2]


def _result(with_poles):
    from nbodykit_b200.binned_statistic import BinnedStatistic
    e = np.array([0.1, 0.2, 0.3, 0.4])
    tri = bs.shell_triples(e)
    rows = bs.pole_triples(e)
    Tsum = np.arange(1, len(tri) + 1) * 64.
    d = bs.bispectrum_table(e, [0.15, 0.25, 0.35], tri, np.arange(len(tri), dtype='f8'), Tsum, 2., 64.)
    power = np.zeros(3, dtype=[('k', 'f8'), ('power', 'c16'), ('modes', 'i8')])
    power['k'] = [0.15, 0.25, 0.35]
    attrs = dict(Nmesh=np.array([4, 4, 4]), BoxSize=np.array([2., 2., 2.]), volume=8., dk=0.1, kmin=0.1, kmax=None,
                 N1=10, shotnoise=0.8, transforms=8 if with_poles else 6, poles=[0, 2] if with_poles else [],
                 los=[0, 0, 1])
    r = object.__new__(bs.FFTBispectrum)
    r.attrs = attrs
    r.comm = SelfComm()
    r.bispec = BinnedStatistic(['k1', 'k2', 'k3'], [e] * 3, d, **attrs)
    r.power = BinnedStatistic(['k'], [e], power, fields_to_sum=['modes'], **attrs)
    r.poles = None
    if with_poles:
        p = bs.poles_table(d, tri, rows, {2: np.linspace(-1, 1, len(rows))}, Tsum, 2., [0, 2])
        r.poles = BinnedStatistic(['k1', 'k2', 'k3'], [e] * 3, p, **attrs)
    return r


@pytest.mark.parametrize("with_poles", [True, False])
def test_save_load_round_trip(tmp_path, with_poles):
    r = _result(with_poles)
    out = str(tmp_path / "bispec.json")
    r.save(out)
    json.load(open(out))
    s = bs.FFTBispectrum.load(out, comm=SelfComm())
    np.testing.assert_array_equal(s.bispec['B'], r.bispec['B'])
    assert s.attrs['poles'] == r.attrs['poles'] and s.attrs['transforms'] == r.attrs['transforms']
    if with_poles:
        assert s.poles.dims == ['k1', 'k2', 'k3']
        for f in ('B_0', 'B_2', 'triangles', 'k1'):
            np.testing.assert_array_equal(s.poles[f], r.poles[f])          # NaN in the same places
    else:
        assert s.poles is None


def test_load_result_saved_without_poles_key(tmp_path):
    """a result saved before multipoles existed (no 'poles' in its state) still loads"""
    r = _result(False)
    state = r.__getstate__()
    del state['poles']
    from nbodykit_b200.utils import JSONEncoder
    out = str(tmp_path / "old.json")
    with open(out, "w") as f:
        json.dump(state, f, cls=JSONEncoder)
    s = bs.FFTBispectrum.load(out, comm=SelfComm())
    assert s.poles is None
    np.testing.assert_array_equal(s.bispec['triangles'], r.bispec['triangles'])


def test_pole_fill_chunks():
    """one fill of the weighted fields writes contiguous shells that miss the same families, at most fill_n slabs"""
    n = 10
    fields = [1 * n + s for s in range(n)] + [2 * n + s for s in range(n)]
    chunks = bs._pole_chunks(fields, n, 4)
    assert chunks == [([1, 2], [2 * i, 2 * i + 1]) for i in range(5)]
    # one family only (the one-family-at-a-time path), with a gap
    assert bs._pole_chunks([2 * n + s for s in (0, 1, 2, 3, 4, 7)], n, 4) == [([2], [0, 1, 2, 3]), ([2], [4]), ([2], [7])]
    # more families than scratch slabs
    assert bs._pole_chunks([f * n + 3 for f in (1, 2, 3, 4)], n, 3) == [([1, 2, 3], [3]), ([4], [3])]
    covered = sorted(f * n + s for fams, run in chunks for f in fams for s in run)
    assert covered == sorted(fields)
