"""RedshiftHistogram argument errors, attributes, the golden fixtures and the oracle's test_with_zhist norms, decided before
any device work (no GPU needed)."""
import os
import pickle

import numpy as np
import pytest

from nbodykit_b200.algorithms import zhist
from nbodykit_b200.comm import SelfComm
from nbodykit_b200.cosmology import Planck15
from nbodykit_b200.lab import ArrayCatalog, RedshiftHistogram
from oracle import zhist_oracle as zo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _cat(z, **cols):
    return ArrayCatalog(dict(z=np.asarray(z, dtype="f8"), **cols), comm=SelfComm())


def _init(cat, *args, **kw):
    """RedshiftHistogram.__init__ without the device passes (explicit edges only)"""
    obj = RedshiftHistogram.__new__(RedshiftHistogram)
    obj._run = lambda z: None
    RedshiftHistogram.__init__(obj, cat, *args, **kw)
    return obj


def _moments(monkeypatch, m):
    """replace the device moments pass with fixed (count, mean, M2, min, max, non-finite)"""
    monkeypatch.setattr(zhist, "local_moments", lambda z: tuple(float(v) for v in m))
    monkeypatch.setattr(zhist, "_column", lambda source, name, dev: np.zeros(0))


def test_missing_columns():
    with pytest.raises(ValueError, match="'Redshift' column missing from input source in RedshiftHistogram"):
        RedshiftHistogram(_cat([0.5]), 1.0, Planck15)
    with pytest.raises(ValueError, match="'W' column missing from input source in RedshiftHistogram"):
        RedshiftHistogram(_cat([0.5]), 1.0, Planck15, redshift="z", weight="W")


@pytest.mark.parametrize("fsky", [0.0, -0.1, np.nan, np.inf, "0.1", [0.1]])
def test_bad_fsky(fsky):
    with pytest.raises(ValueError, match="fsky"):
        RedshiftHistogram(_cat([0.5]), fsky, Planck15, redshift="z", bins=[0.1, 0.2])


def test_cosmo_needs_comoving_distance():
    with pytest.raises(ValueError, match="comoving_distance"):
        RedshiftHistogram(_cat([0.5]), 1.0, object(), redshift="z", bins=[0.1, 0.2])


@pytest.mark.parametrize("bins", [[0.1], [], [[0.1, 0.2], [0.3, 0.4]], [0.1, np.nan, 0.3], [0.1, np.inf],
                                  [0.2, 0.1], [0.1, 0.1, 0.2], [-1.0, 0.1], [-2.0, -1.5], ["a", "b"]])
def test_bad_edges(bins):
    with pytest.raises(ValueError, match="edges"):
        RedshiftHistogram(_cat([0.5]), 1.0, Planck15, redshift="z", bins=bins)


@pytest.mark.parametrize("bins", [0, -3, 2.5, True])
def test_bad_int_bins(bins):
    with pytest.raises(ValueError, match="positive integer"):
        RedshiftHistogram(_cat([0.5]), 1.0, Planck15, redshift="z", bins=bins)


@pytest.mark.parametrize("bins", [None, 10])
@pytest.mark.parametrize("m,match", [((10, 0.5, 0.1, 0.1, 0.9, 1), "non-finite"), ((0, 0, 0, np.inf, -np.inf, 0), "empty"),
                                     ((1, 0.5, 0.0, 0.5, 0.5, 0), "zero spread"), ((5, 0.5, 0.0, 0.5, 0.5, 0), "zero spread")])
def test_scott_and_int_bins_refuse_bad_redshifts(monkeypatch, bins, m, match):
    _moments(monkeypatch, m)
    with pytest.raises(ValueError, match=match):
        RedshiftHistogram(_cat([0.5]), 1.0, Planck15, redshift="z", bins=bins)


def test_scott_edges_from_merged_moments(monkeypatch):
    """the edges are built on the host from the reduced statistics, as the oracle builds them"""
    z = zo.make_redshifts(42, 1000)
    n = z.size
    mean = z.sum() / n
    _moments(monkeypatch, (n, mean, ((z - mean) ** 2).sum(), z.min(), z.max(), 0))
    h, edges = zhist.scotts_bin_width(np.zeros(0), SelfComm())
    want_h, want = zo.scott_edges(z)
    np.testing.assert_allclose(edges, want, rtol=1e-13, atol=0)
    assert len(edges) == len(want)


def test_chan_merge_in_rank_order():
    rng = np.random.RandomState(3)
    parts = [rng.normal(0.5, 0.1, k) for k in (5, 0, 17, 1)]

    def state(a):
        if a.size == 0:
            return (0.0, 0.0, 0.0, np.inf, -np.inf, 0.0)
        m = a.mean()
        return (float(a.size), m, ((a - m) ** 2).sum(), a.min(), a.max(), 0.0)
    m = state(parts[0])
    for p in parts[1:]:
        m = zhist._merge(m, state(p))
    z = np.concatenate(parts)
    assert m[0] == z.size and m[3] == z.min() and m[4] == z.max()
    np.testing.assert_allclose(m[1], z.mean(), rtol=1e-15)
    np.testing.assert_allclose(m[2], ((z - z.mean()) ** 2).sum(), rtol=1e-13)


def test_attrs_and_state():
    r = _init(_cat([0.5], W=[1.0]), 0.25, Planck15, bins=[0.1, 0.3, 0.7], redshift="z", weight="W")
    assert r.attrs["fsky"] == 0.25 and r.attrs["redshift"] == "z" and r.attrs["weight"] == "W"
    assert r.attrs["cosmo"] == Planck15.pars
    np.testing.assert_array_equal(r.attrs["edges"], [0.1, 0.3, 0.7])
    assert r.attrs["edges"].dtype == np.float64
    mapping = _init(_cat([0.5]), 1.0, zo_cosmo_dict(), bins=[0.1, 0.2], redshift="z")
    assert mapping.attrs["cosmo"] == dict(Planck15.pars)


def zo_cosmo_dict():
    class D(dict):
        def comoving_distance(self, z):
            return Planck15.comoving_distance(z)
    return D(Planck15.pars)


@pytest.mark.parametrize("ext", ["nearest", 4, -1, None, 1.5])
def test_ext_names(ext):
    r = RedshiftHistogram.__new__(RedshiftHistogram)
    with pytest.raises(ValueError, match="Unknown extrapolation mode"):
        r.interpolate(np.zeros(3), ext=ext)


def test_fewer_than_four_bins_cannot_interpolate():
    r = RedshiftHistogram.__new__(RedshiftHistogram)
    r.bin_centers, r.nbar = np.array([0.1, 0.2, 0.3]), np.ones(3)
    with pytest.raises(ValueError, match="at least 4 bins"):
        r.interpolate(np.zeros(3))


def test_even_edges_detection():
    assert zhist._inverse_width(0.1 + 0.01 * np.arange(11)) == pytest.approx(100.)
    assert zhist._inverse_width(np.linspace(0.2, 0.9, 50)) == pytest.approx(49 / 0.7)
    assert zhist._inverse_width(np.array([0.1, 0.2, 0.25, 0.4])) == 0.0


def test_golden_fixtures_load():
    """the reference's output: edges, nbar, interpolation, and a file of its save()"""
    for name in ("scott", "explicit"):
        g = np.load(os.path.join(GOLDEN, "zhist_%s.npz" % name))
        bins = None if name == "scott" else g["bin_edges"]
        o = zo.zhist(g["z"], float(g["fsky"]), Planck15, bins=bins)
        np.testing.assert_array_equal(o["bin_edges"], g["bin_edges"])
        np.testing.assert_array_equal(o["nbar"], g["nbar"])
        np.testing.assert_allclose(zo.zhist(g["z"], float(g["fsky"]), Planck15, bins=bins, w=g["w"])["nbar"],
                                   g["nbar_weighted"], rtol=1e-14)
        for e in ("extrapolate", "zeros", "const"):
            np.testing.assert_array_equal(zo.interpolate(g["x"], g["bin_centers"], g["nbar"], e), g["interp_%s" % e])
    r = RedshiftHistogram.load(os.path.join(GOLDEN, "zhist_reference_save.json"), comm=SelfComm())
    g = np.load(os.path.join(GOLDEN, "zhist_scott.npz"))
    for k in ("bin_edges", "bin_centers", "dV", "nbar"):
        np.testing.assert_array_equal(getattr(r, k), g[k])
    assert r.attrs["fsky"] == float(g["fsky"]) and r.attrs["cosmo"] == Planck15.pars


def test_pickle_round_trip():
    r = RedshiftHistogram.__new__(RedshiftHistogram)
    r.__setstate__(dict(bin_edges=np.arange(3.), bin_centers=np.array([0.5, 1.5]), dV=np.ones(2), nbar=np.ones(2),
                        attrs=dict(edges=np.arange(3.), fsky=1.0, redshift="z", weight=None, cosmo=None)))
    r2 = pickle.loads(pickle.dumps(r))
    assert sorted(r2.__dict__) == sorted(r.__getstate__())
    np.testing.assert_array_equal(r2.nbar, r.nbar)


def test_with_zhist_norms_from_the_oracle():
    """the reference's test_conv_power.py::test_with_zhist constants from this package's streams and Planck15"""
    data_norm, randoms_norm, _, _ = zo.with_zhist_norms()
    np.testing.assert_allclose(data_norm, zo.DATA_NORM, rtol=1e-4)
    np.testing.assert_allclose(randoms_norm, zo.RANDOMS_NORM, rtol=1e-4)
    assert abs(data_norm / zo.DATA_NORM - 1) < 3e-5 and abs(randoms_norm / zo.RANDOMS_NORM - 1) < 3e-5


def test_exported_from_lab():
    import nbodykit_b200.lab as lab
    assert lab.RedshiftHistogram is RedshiftHistogram and "RedshiftHistogram" in lab.__dict__
