"""oracle/zhist_oracle.py pinned against the reference's own RedshiftHistogram (nbodykit/algorithms/zhist.py run verbatim
on one rank by oracle/zhist_refload.py): Scott's edges and counts, weighted and unweighted, rows on interior edges, on the
last edge, below the first edge and NaN under explicit edges, `interpolate` in all four extrapolation modes, and the JSON
files of `save` read both ways.  Skipped where the reference tree is absent."""
import json
import warnings

import numpy as np
import pytest

from oracle import zhist_oracle as zo, zhist_refload

pytestmark = pytest.mark.skipif(not zhist_refload.available(), reason="reference tree not present")

FSKY = 0.15


def _cosmo():
    from nbodykit_b200.cosmology import Planck15
    return Planck15


def _ref(z, bins=None, w=None):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return zhist_refload.run(z, FSKY, zhist_refload.CosmoDict(_cosmo()), bins=bins, w=w)


def _mine(z, bins=None, w=None):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return zo.zhist(z, FSKY, _cosmo(), bins=bins, w=w)


@pytest.mark.parametrize("n,seed", [(1000, 42), (10000, 84), (2, 1), (37, 3)])
@pytest.mark.parametrize("weighted", [False, True])
def test_scott_edges_and_counts(n, seed, weighted):
    z = zo.make_redshifts(seed, n)
    w = np.random.RandomState(seed).uniform(size=n) if weighted else None
    r, o = _ref(z, w=w), _mine(z, w=w)
    np.testing.assert_array_equal(o["bin_edges"], r.bin_edges)
    np.testing.assert_array_equal(o["bin_centers"], r.bin_centers)
    np.testing.assert_array_equal(o["dV"], r.dV)
    np.testing.assert_array_equal(o["nbar"], r.nbar)
    if not weighted:
        assert (r.nbar * r.dV).sum() == n or o["N"].sum() < n      # the maximum may sit on the last edge


def test_float32_redshifts_are_widened_exactly():
    """the contract widens float32 redshifts to float64 first: the reference's answer on the widened column.  On the
    float32 column itself the reference sums Scott's statistics in float32, and its edges move by about 1e-8"""
    z = zo.make_redshifts(5, 3000).astype("f4")
    r, o = _ref(z.astype("f8")), _mine(z)
    np.testing.assert_array_equal(o["bin_edges"], r.bin_edges)
    np.testing.assert_array_equal(o["nbar"], r.nbar)
    np.testing.assert_allclose(_ref(z).bin_edges, r.bin_edges, rtol=1e-6)


@pytest.mark.parametrize("weighted", [False, True])
def test_explicit_edges_rows_on_edges_outside_and_nan(weighted):
    edges = np.array([0.1, 0.2, 0.25, 0.4, 0.45, 0.5, 0.55, 0.62, 0.8, 1.0])
    rng = np.random.RandomState(11)
    z = np.concatenate([rng.uniform(0.0, 1.1, 500), edges, edges, [np.nan, 0.05, 1.0, 1.5, np.nextafter(1.0, 0)]])
    w = rng.uniform(size=z.size) if weighted else None
    r, o = _ref(z, bins=edges, w=w), _mine(z, bins=edges, w=w)
    np.testing.assert_array_equal(o["nbar"], r.nbar)
    # every edge but the last counts its row in the bin above it; the last edge, NaN and the rows outside count nowhere
    n_in = ((z >= edges[0]) & (z < edges[-1])).sum()
    if not weighted:
        assert o["N"].sum() == n_in
        assert o["N"][0] == ((z >= 0.1) & (z < 0.2)).sum()


@pytest.mark.parametrize("ext", ["extrapolate", "zeros", "raise", "const", 0, 1, 2, 3])
def test_interpolate_all_modes(ext):
    z = zo.make_redshifts(42, 1000)
    r, o = _ref(z), _mine(z)
    c = o["bin_centers"]
    inside = np.linspace(c[0], c[-1], 201)
    outside = np.array([c[0] - 0.1, c[-1] + 0.05, -0.5, 2.0])
    if zo.EXT[ext] == 2:
        np.testing.assert_array_equal(zo.interpolate(inside, c, o["nbar"], ext), r.interpolate(inside, ext))
        with pytest.raises(ValueError):
            r.interpolate(outside, ext)
        with pytest.raises(ValueError):
            zo.interpolate(outside, c, o["nbar"], ext)
        assert zo.splev(outside, *zo.spline(c, o["nbar"]), ext)[1] == len(outside)
        return
    x = np.concatenate([inside, outside, c])
    want = r.interpolate(x, ext)
    np.testing.assert_array_equal(zo.interpolate(x, c, o["nbar"], ext), want)
    # the restated splev, the evaluation the kernel performs
    got, nout = zo.splev(x, *zo.spline(c, o["nbar"]), ext)
    np.testing.assert_array_equal(got, want)
    assert nout == len(outside)


def test_save_files_read_both_ways(tmp_path):
    """a file written by the reference's save() loads in this package, and one written here loads in the reference"""
    from nbodykit_b200.algorithms.zhist import RedshiftHistogram
    from nbodykit_b200.comm import SelfComm
    z = zo.make_redshifts(42, 1000)
    r = _ref(z)
    path = str(tmp_path / "ref.json")
    r.save(path)
    mine = RedshiftHistogram.load(path, comm=SelfComm())
    for k in ("bin_edges", "bin_centers", "dV", "nbar"):
        np.testing.assert_array_equal(getattr(mine, k), getattr(r, k))
    assert mine.attrs["fsky"] == FSKY and mine.attrs["redshift"] == "z" and mine.attrs["weight"] is None
    assert mine.attrs["cosmo"] == dict(_cosmo().pars)
    np.testing.assert_array_equal(mine.attrs["edges"], r.attrs["edges"])

    # written here (the same state dictionary, through this package's JSONEncoder), read by the reference
    obj = RedshiftHistogram.__new__(RedshiftHistogram)
    obj.__setstate__(dict(bin_edges=r.bin_edges, bin_centers=r.bin_centers, dV=r.dV, nbar=r.nbar,
                          attrs=dict(edges=r.attrs["edges"], fsky=FSKY, redshift="z", weight=None, cosmo=dict(_cosmo().pars))))
    obj.comm = SelfComm()
    path2 = str(tmp_path / "mine.json")
    obj.save(path2)
    back = zhist_refload.load_saved(path2)
    for k in ("bin_edges", "bin_centers", "dV", "nbar"):
        np.testing.assert_array_equal(getattr(back, k), getattr(r, k))
    assert sorted(json.load(open(path2))) == sorted(json.load(open(path)))
    np.testing.assert_array_equal(back.interpolate(r.bin_centers), r.interpolate(r.bin_centers))


def test_int_bins_raise_name_error_in_the_reference():
    """the reference's int-bins branch calls an unimported `linspace`; this package implements its docstring"""
    z = zo.make_redshifts(42, 100)
    with pytest.raises(NameError):
        _ref(z, bins=10)
    o = _mine(z, bins=10)
    np.testing.assert_array_equal(o["bin_edges"], np.linspace(z.min(), z.max(), 11))
    assert o["N"].sum() == (z < z.max()).sum()
