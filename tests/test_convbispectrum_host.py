"""ConvolvedFFTBispectrum without a GPU: the oracle's FFT form (Y_lm, r2c, shell c2r) equals its FFT-free direct form
(explicit L_ell sums, closed triangles); the arguments are refused before any device work; the row and table layout;
save / load."""
import numpy as np
import pytest

import convbispectrum_oracle as cbo


def _fields(N, seed):
    L = np.array([300., 260., 240.])
    C = np.array([40., -500., 900.])
    rng = np.random.RandomState(seed)
    nd, nr = 60, 240
    dpos = rng.uniform(-0.5, 0.5, (nd, 3)) * L + C
    rpos = rng.uniform(-0.5, 0.5, (nr, 3)) * L + C
    d = dict(wc=rng.uniform(.8, 1.2, nd), wf=rng.uniform(.5, 1, nd), nbar=np.full(nd, 1e-4), v=rng.uniform(.9, 1.1, nd))
    r = dict(wc=np.ones(nr), wf=rng.uniform(.5, 1, nr), nbar=np.full(nr, 1e-4), v=np.ones(nr))
    return L, C, cbo.fkp_fields(dpos, rpos, d, r, N, L, C, "cic")


@pytest.mark.parametrize("N", [(12, 12, 12), (16, 12, 10)])
def test_fft_form_equals_direct_form(N):
    L, C, f = _fields(N, 1)
    kedges = np.arange(0, np.pi * min(N) / L.max() + 0.02, 2 * np.pi / L.min())
    args = (f["F"], f["N"], N, L, C, kedges, [0, 2, 4], "CompensateCICShotnoise", f["randoms_norm3"], f["S3"])
    a, b = cbo.fft_form(*args), cbo.direct_form(*args)
    np.testing.assert_array_equal(a["triangles"], b["triangles"])
    np.testing.assert_array_equal(a["row_triangles"], b["row_triangles"])
    ok = a["row_triangles"] > 0
    assert ok.sum() > 5
    for ell in (0, 2, 4):
        assert np.isnan(b["B_%d" % ell][~ok]).all()
        assert (np.abs(a["B_%d" % ell] - b["B_%d" % ell])[ok] <= 1e-12 * a["bound_%d" % ell][ok]).all(), ell
    okt = a["triangles"] > 0
    assert (np.abs(a["shotnoise_0"] - b["shotnoise_0"])[okt] <= 1e-12 * a["shot_bound"][okt]).all()


@pytest.mark.parametrize("poles", [[1], [0, 3], [0, 0], [10], [0, 2.5], []])
def test_bad_poles_raise_before_device_work(poles):
    from nbodykit_b200.lab import ConvolvedFFTBispectrum
    with pytest.raises(ValueError):
        ConvolvedFFTBispectrum(None, poles=poles)        # refused before the mesh is even looked at


def test_bad_shells_raise_before_device_work(monkeypatch):
    """dk = 0 and kmin < 0 are refused from the mesh geometry alone: no paint and no transform runs"""
    from nbodykit_b200.algorithms import convbispectrum as cb
    from nbodykit_b200.algorithms.convpower.catalogmesh import FKPCatalogMesh

    class Geometry(FKPCatalogMesh):
        attrs = dict(Nmesh=np.array([16, 16, 16]), BoxSize=np.array([100.] * 3), BoxCenter=np.zeros(3), BoxPad=0.02)
        resampler, interlaced, comm = 'cic', False, None

        def __init__(self):
            pass

        def compute(self, *a, **k):
            raise AssertionError("painted")

    monkeypatch.setattr(cb.ConvolvedFFTBispectrum, "run", lambda self: pytest.fail("ran"))
    for kw in (dict(dk=0.), dict(kmin=-1.), dict(dk=0.01, kmax=0.02, kmin=0.015)):
        with pytest.raises(ValueError):
            cb.ConvolvedFFTBispectrum(Geometry(), poles=[0], **kw)
    with pytest.raises(TypeError):
        cb.ConvolvedFFTBispectrum(object(), poles=[0])


def test_table_layout():
    """B_0 and shotnoise_0 fill every permutation of a sorted triple, B_ell the (b, c) pair of each row; the shot sum
    counts a shell once per occurrence in its triple"""
    from nbodykit_b200.algorithms.bispectrum import pole_triples, shell_triples
    from nbodykit_b200.algorithms.convbispectrum import convolved_table
    kedges = np.array([0., 1., 2., 3.])
    tri, rows = shell_triples(kedges), pole_triples(kedges)
    n = 3
    Nc = 8
    Tsum = np.full(len(tri), 2. * Nc)                # two triangles each
    S = np.arange(1., len(tri) + 1)
    W = {2: np.arange(1., len(rows) + 1)}
    Hsum = np.ones(len(rows))
    V, I33, S3 = 2., 4., 0.5
    d = convolved_table(kedges, np.array([.5, 1.5, 2.5]), tri, rows, S, W, Tsum, Hsum, V, I33, S3, Nc, [0, 2])
    assert d.dtype.names == ('k1', 'k2', 'k3', 'B_0', 'B_2', 'shotnoise_0', 'triangles')
    for q, (i, j, l) in enumerate(tri.tolist()):
        for p in {(i, j, l), (l, j, i), (j, l, i)}:
            assert d['triangles'][p] == 2
            assert d['B_0'][p] == V ** 3 * S[q] / (I33 * Tsum[q])
            # the rows of the triple carry its distinct shells; with their multiplicities they sum three H terms
            assert np.isclose(d['shotnoise_0'][p], (3 / Tsum[q] - 2 * S3) / I33)
    for q, (a, b, c) in enumerate(rows.tolist()):
        t = [k for k, x in enumerate(tri.tolist()) if x == sorted([a, b, c])][0]
        assert d['B_2'][a, b, c] == d['B_2'][a, c, b] == V ** 3 * W[2][q] / (I33 * Tsum[t])
    missing = d['triangles'] == 0
    assert missing.any() and np.isnan(d['B_0'][missing]).all() and np.isnan(d['B_2'][missing]).all()
    assert np.isnan(d['shotnoise_0'][missing]).all()
    assert d['k1'][2, 0, 0] == 2.5 and d['k3'][0, 0, 1] == 1.5 and d.shape == (n, n, n)


def test_save_load_round_trip(tmp_path):
    from nbodykit_b200.algorithms.bispectrum import pole_triples, shell_triples
    from nbodykit_b200.algorithms.convbispectrum import ConvolvedFFTBispectrum, convolved_table
    from nbodykit_b200.binned_statistic import BinnedStatistic
    from nbodykit_b200.comm import SelfComm
    kedges = np.array([0., 1., 2., 3.])
    tri, rows = shell_triples(kedges), pole_triples(kedges)
    d = convolved_table(kedges, np.array([.5, 1.5, 2.5]), tri, rows, np.ones(len(tri)), {2: np.ones(len(rows))},
                        np.full(len(tri), 8.), np.ones(len(rows)), 2., 1., 0., 8, [0, 2])
    r = object.__new__(ConvolvedFFTBispectrum)
    r.comm = SelfComm()
    r.edges = kedges
    r.attrs = dict(poles=[0, 2], dk=1., kmin=0., kmax=None, Nmesh=np.array([8, 8, 8]), BoxSize=np.ones(3),
                   alpha=0.1, S3=2.5, transforms=30, **{'data.norm3': 1., 'randoms.norm3': 1.02})
    r.poles = BinnedStatistic(['k1', 'k2', 'k3'], [kedges] * 3, d, **r.attrs)
    path = str(tmp_path / "cb.json")
    r.save(path)
    s = ConvolvedFFTBispectrum.load(path, comm=SelfComm())
    np.testing.assert_array_equal(s.edges, kedges)
    assert s.poles.dims == ['k1', 'k2', 'k3']
    for f in d.dtype.names:
        np.testing.assert_array_equal(s.poles[f], r.poles[f])
    assert s.attrs['poles'] == [0, 2] and s.attrs['S3'] == 2.5 and s.attrs['randoms.norm3'] == 1.02
    np.testing.assert_array_equal(s.attrs['Nmesh'], [8, 8, 8])
