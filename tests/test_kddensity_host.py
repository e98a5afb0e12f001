"""KDDensity argument errors and attributes, decided before any device work (no GPU needed)."""
import numpy as np
import pytest

from nbodykit_b200.algorithms import kdtree
from nbodykit_b200.comm import SelfComm
from nbodykit_b200.lab import ArrayCatalog, KDDensity


def _cat(n=20, **attrs):
    rng = np.random.RandomState(0)
    return ArrayCatalog({"Position": rng.uniform(size=(n, 3)) * 10, "m": rng.uniform(size=n)}, comm=SelfComm(), **attrs)


def _init(cat, **kw):
    """KDDensity.__init__ without the device run"""
    obj = KDDensity.__new__(KDDensity)
    obj.run = lambda: None
    KDDensity.__init__(obj, cat, **kw)
    return obj


def test_reference_errors():
    with pytest.raises(ValueError, match="'Position' column"):
        KDDensity(ArrayCatalog({"m": np.ones(3)}, comm=SelfComm(), BoxSize=1.))
    with pytest.raises(ValueError, match="'BoxSize' in the input source 'attrs'"):
        KDDensity(_cat())


@pytest.mark.parametrize("box", [[10., 10., 11.], [1., 2., 3.]])
def test_non_cubic_box(box):
    with pytest.raises(ValueError, match="cubic"):
        KDDensity(_cat(BoxSize=np.array(box)))


@pytest.mark.parametrize("box", [[10., 10.], np.ones((3, 3)), [0., 0., 0.], [-1., -1., -1.], [np.inf] * 3])
def test_bad_box(box):
    with pytest.raises(ValueError, match="BoxSize"):
        KDDensity(_cat(BoxSize=np.array(box)))


@pytest.mark.parametrize("margin", [-1., np.nan, np.inf, [1., 2.]])
def test_bad_margin(margin):
    with pytest.raises(ValueError, match="margin"):
        KDDensity(_cat(BoxSize=10.), margin=margin)


@pytest.mark.parametrize("box", [10., [10.], np.array([10.]), np.float32(10.)])
def test_boxsize_broadcast_and_attrs(box):
    r = _init(_cat(n=20, BoxSize=box), margin=0.5)
    assert r.attrs["BoxSize"].dtype == np.float64 and r.attrs["BoxSize"].shape == (3,)
    np.testing.assert_array_equal(r.attrs["BoxSize"], [10.] * 3)
    assert r.attrs["margin"] == 0.5
    assert r.attrs["meansep"] == (20 / 1000.) ** (1 / 3.)


def test_margin_is_stored_as_given():
    r = _init(_cat(BoxSize=10.), margin=3)
    assert r.attrs["margin"] == 3 and isinstance(r.attrs["margin"], int)
    assert _init(_cat(BoxSize=10.)).attrs["margin"] == 1.0


def test_too_many_rows_on_one_rank(monkeypatch):
    cat = _cat(BoxSize=10.)
    monkeypatch.setattr(type(cat), "size", property(lambda self: 1 << 31))
    with pytest.raises(ValueError, match="2\\^31"):
        KDDensity(cat)


def test_cells_follow_the_global_row_count():
    assert kdtree._ncell(0) == [1, 1, 1] and kdtree._ncell(7) == [1, 1, 1]
    n = kdtree._ncell(10 ** 6)[0]
    assert n ** 3 * kdtree._ROWS_PER_CELL <= 10 ** 6 < (n + 1) ** 3 * kdtree._ROWS_PER_CELL
    assert kdtree._ncell(10 ** 12) == [kdtree._MAX_CELLS_PER_AXIS] * 3


def test_exported_from_lab():
    import nbodykit_b200.lab as lab
    assert lab.KDDensity is KDDensity and "KDDensity" in lab.__dict__
