"""FFTBispectrum host logic without a GPU: argument validation, the shell triples and their closure rule, the symmetric
table with NaN where no triangle is evaluated, save/load, and the float64 oracle's FFT form against its FFT-free direct
sum."""
import json

import numpy as np
import pytest

from nbodykit_b200.algorithms import bispectrum as bs
from nbodykit_b200.comm import SelfComm
from oracle import bispectrum_oracle as bo


def test_dk_zero_raises():
    with pytest.raises(ValueError, match="dk = 0"):
        bs.shell_edges(32, 100., dk=0.)
    with pytest.raises(ValueError, match="dk > 0"):
        bs.shell_edges(32, 100., dk=-0.1)
    with pytest.raises(ValueError, match="kmin"):
        bs.shell_edges(32, 100., kmin=-0.1)
    with pytest.raises(ValueError, match="no k shell"):
        bs.shell_edges(32, 100., kmin=10.)


def test_shell_limit():
    m = bs.max_shells()
    assert m >= 64
    L = 100.
    dk = 0.01
    e = bs.shell_edges(1024, L, dk=dk, kmax=(m + 0.5) * dk)
    assert len(e) - 1 == m
    with pytest.raises(ValueError, match="maximum of %d" % m):
        bs.shell_edges(1024, L, dk=dk, kmax=(m + 1.5) * dk)


def test_edges_follow_fftpower():
    N, L = np.array([32, 24, 16]), np.array([100., 80., 60.])
    dk = 2 * np.pi / L.min()
    kmax = np.pi * N.min() / L.max() + dk / 2
    np.testing.assert_array_equal(bs.shell_edges(N, L), np.arange(0., kmax, dk))
    np.testing.assert_array_equal(bs.shell_edges(N, L, dk=0.05, kmin=0.02, kmax=0.4), np.arange(0.02, 0.4, 0.05))


def test_triples_closure_rule():
    e = np.array([0., 1., 2., 3., 4., 5.])
    t = bs.shell_triples(e)
    want = [(i, j, l) for i in range(5) for j in range(i, 5) for l in range(j, 5) if e[l] < e[i + 1] + e[j + 1]]
    assert [tuple(r) for r in t] == want
    assert (0, 0, 1) in want and (0, 0, 2) not in want and (0, 1, 2) in want and (1, 1, 3) in want and (1, 1, 4) not in want
    assert t.dtype == np.int32
    np.testing.assert_array_equal(t, bo.triples(e))
    # non-zero kmin shifts the rule with the edges
    e2 = e + 0.5
    assert [tuple(r) for r in bs.shell_triples(e2)] == [tuple(r) for r in bo.triples(e2)]


def test_table_symmetric_and_nan():
    e = np.array([0., 0.1, 0.2, 0.3])
    tri = bs.shell_triples(e)
    rng = np.random.RandomState(3)
    N3 = 1000.
    counts = rng.randint(0, 5, size=len(tri))
    counts[0] = 0
    Tsum = counts * N3
    S = rng.normal(size=len(tri))
    kmean = np.array([0.15, 0.25, 0.35])
    d = bs.bispectrum_table(e, kmean, tri, S, Tsum, 8.0, N3)
    assert d.shape == (3, 3, 3)
    assert d['B'].dtype == np.float64 and d['triangles'].dtype == np.int64
    for (i, j, l), c, s in zip(tri, counts, S):
        for p in [(i, j, l), (i, l, j), (j, i, l), (j, l, i), (l, i, j), (l, j, i)]:
            assert d['triangles'][p] == c
            if c:
                assert d['B'][p] == 64.0 * s / (c * N3)
    assert (np.isnan(d['B']) == (d['triangles'] == 0)).all()
    # (0, 0, 2) fails the closure rule: never evaluated
    assert d['triangles'][0, 0, 2] == 0 and np.isnan(d['B'][2, 0, 0])
    np.testing.assert_array_equal(d['k1'][:, 0, 0], kmean)
    np.testing.assert_array_equal(d['k3'][0, 0, :], kmean)


def test_save_load_round_trip(tmp_path):
    from nbodykit_b200.binned_statistic import BinnedStatistic
    e = np.array([0.1, 0.2, 0.3, 0.4])
    tri = bs.shell_triples(e)
    d = bs.bispectrum_table(e, [0.15, 0.25, 0.35], tri, np.arange(len(tri), dtype='f8'), np.arange(len(tri)) * 64., 2.,
                            64.)
    power = np.zeros(3, dtype=[('k', 'f8'), ('power', 'c16'), ('modes', 'i8')])
    power['k'] = [0.15, 0.25, 0.35]
    power['power'] = [1 + 0j, 2, 3]
    power['modes'] = [6, 18, 30]
    attrs = dict(Nmesh=np.array([4, 4, 4]), BoxSize=np.array([2., 2., 2.]), volume=8., dk=0.1, kmin=0.1, kmax=None, N1=10,
                 shotnoise=0.8, transforms=6)
    r = object.__new__(bs.FFTBispectrum)
    r.attrs = attrs
    r.comm = SelfComm()
    r.bispec = BinnedStatistic(['k1', 'k2', 'k3'], [e] * 3, d, **attrs)
    r.power = BinnedStatistic(['k'], [e], power, fields_to_sum=['modes'], **attrs)
    out = str(tmp_path / "bispec.json")
    r.save(out)
    json.load(open(out))
    s = bs.FFTBispectrum.load(out, comm=SelfComm())
    assert s.bispec.dims == ['k1', 'k2', 'k3']
    np.testing.assert_array_equal(s.bispec['triangles'], d['triangles'])
    np.testing.assert_array_equal(s.bispec['B'], d['B'])           # NaN in the same places
    np.testing.assert_array_equal(s.power['power'], power['power'])
    assert s.attrs['transforms'] == 6 and s.attrs['shotnoise'] == 0.8


@pytest.mark.parametrize("N,L", [((12, 12, 12), (100., 100., 100.)), ((15, 15, 15), (80., 80., 80.)),
                                 ((16, 12, 10), (100., 70., 60.))], ids=["12", "15-odd", "16x12x10"])
def test_oracle_fft_form_equals_direct_sum(N, L):
    rng = np.random.RandomState(7)
    half = np.fft.rfftn(rng.normal(size=N) + 0.3 * rng.normal(size=N) ** 2) / np.prod(N)
    dk = 2 * np.pi / min(L)
    kedges = np.arange(0., np.pi * min(N) / max(L) + dk / 2, dk)
    a = bo.fft_form(half, N, L, kedges)
    b = bo.direct_form(half, N, L, kedges)
    np.testing.assert_array_equal(a['triangles'], b['triangles'])
    ok = a['triangles'] > 0
    assert ok.sum() > 5
    np.testing.assert_array_equal(np.isnan(a['B']), ~ok)
    assert (np.abs(a['B'] - b['B'])[ok] <= 1e-12 * a['bound'][ok]).all()
    # the counts are integers in the FFT form too
    assert np.abs(a['Tsum'] / np.prod(N) - a['triangles']).max() < 1e-6
