"""CylindricalGroups and CatalogSource.sort argument errors, raised before any device work (no GPU needed)."""
import numpy as np
import pytest

from nbodykit_b200.comm import SelfComm
from nbodykit_b200.lab import ArrayCatalog, CylindricalGroups


def _cat(n=20, box=True):
    rng = np.random.RandomState(0)
    kw = dict(BoxSize=np.array([10., 10., 10.])) if box else {}
    return ArrayCatalog({"Position": rng.uniform(size=(n, 3)) * 10, "m": rng.uniform(size=n), "s": np.array(["a"] * n),
                         "v": rng.uniform(size=(n, 2))}, comm=SelfComm(), **kw)


def test_reference_errors():
    cat = _cat()
    with pytest.raises(ValueError, match="no such column"):
        CylindricalGroups(cat, "missing", 1., 1., periodic=True, flat_sky_los=[0, 0, 1])
    with pytest.raises(ValueError, match="length 3"):
        CylindricalGroups(cat, "m", 1., 1., periodic=True, flat_sky_los=[0, 0, 0, 1])
    with pytest.raises(ValueError, match="unit vector"):
        CylindricalGroups(cat, "m", 1., 1., periodic=True, flat_sky_los=[1, 1, 1])
    with pytest.raises(ValueError, match="BoxSize"):
        CylindricalGroups(_cat(box=False), "m", 1., 1., periodic=True, flat_sky_los=[0, 0, 1])
    with pytest.raises(ValueError, match="Position"):
        CylindricalGroups(ArrayCatalog({"m": np.ones(3)}, comm=SelfComm()), "m", 1., 1.)


@pytest.mark.parametrize("rperp,rpar", [(-1., 1.), (1., -1.), (np.inf, 1.), (1., np.nan), (0., 0.)])
def test_bad_radii(rperp, rpar):
    with pytest.raises(ValueError, match="rperp|rpar"):
        CylindricalGroups(_cat(), "m", rperp, rpar, flat_sky_los=[0, 0, 1])


def test_too_many_rows_on_one_rank(monkeypatch):
    cat = _cat()
    monkeypatch.setattr(type(cat), "size", property(lambda self: 1 << 31))
    with pytest.raises(ValueError, match="2\\^31"):
        CylindricalGroups(cat, "m", 1., 1., flat_sky_los=[0, 0, 1])


def test_source_boxsize_wins_over_keyword():
    from nbodykit_b200.algorithms import cgm
    obj = cgm.CylindricalGroups.__new__(cgm.CylindricalGroups)
    obj.run = lambda: None
    cgm.CylindricalGroups.__init__(obj, _cat(), "m", 1., 1., flat_sky_los=[0, 0, 1], BoxSize=3.)
    np.testing.assert_array_equal(obj.attrs["BoxSize"], [10., 10., 10.])
    assert obj.attrs["rankby"] == ["m"] and obj.attrs["rperp"] == 1. and obj.attrs["periodic"] is False


def test_sort_errors_before_device_work():
    cat = _cat()
    with pytest.raises(ValueError, match="duplicated"):
        cat.sort(["m", "m"])
    with pytest.raises(ValueError, match="invalid sort keys"):
        cat.sort(["nope"])
    with pytest.raises(ValueError, match="list or tuple"):
        cat.sort("m", usecols={"m"})
    with pytest.raises(ValueError, match="invalid column names"):
        cat.sort("m", usecols=["nope"])
    with pytest.raises(ValueError, match="integer or floating"):
        cat.sort("s")
    with pytest.raises(ValueError, match="one-dimensional"):
        cat.sort("v")
