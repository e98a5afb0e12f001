"""oracle/fof_oracle.py pinned against the reference's own FOF helpers (nbodykit/algorithms/fof.py: `_assign_labels`,
`centerofmass`, `count`, `fof_catalog`, loaded verbatim by oracle/fof_refload.py).  Without ties among group sizes the
labels are identical and the float64 centres of mass agree to 1e-12 of the box; with ties the partition and the sizes
are identical.  Skipped where the reference tree is absent."""
import numpy as np
import pytest

from oracle import fof_oracle as fo, fof_refload

pytestmark = pytest.mark.skipif(not fof_refload.available(), reason="reference tree not present")


def _same_partition(a, b):
    pairs = set(zip(a.tolist(), b.tolist()))
    return len(pairs) == len(set(a.tolist())) == len(set(b.tolist()))


@pytest.mark.parametrize("name", sorted(fo.fixture_cases()))
def test_oracle_labels_and_features_match_the_reference(name):
    ref = fof_refload.load()
    comm = ref.Comm()
    pos, vel, peak, box, b, nmin = fo.fixture_cases()[name]
    mid = fo.minid(pos, b, box)
    want = np.asarray(ref._assign_labels(mid, comm=comm, thresh=nmin))
    got = fo.labels_from_minid(mid, nmin)
    sizes = np.bincount(want)[1:]
    assert _same_partition(got, want)
    assert sorted(np.bincount(got)[1:]) == sorted(sizes)
    assert np.array_equal(ref.count(want, comm=comm)[1:], sizes)
    if len(np.unique(sizes)) == len(sizes):
        np.testing.assert_array_equal(got, want)
    # features on the same labels: the reference's float64 centerofmass vs the restatement
    pos8, vel8 = pos.astype("f8"), vel.astype("f8")
    scale = np.max(box) if box is not None else np.ptp(pos8)
    mine = fo.features(got, pos8, vel8, box, peak=peak)
    nlab = got.max() + 1
    with np.errstate(invalid="ignore"):
        cm = ref.centerofmass(got, pos8, boxsize=np.asarray(box) if box is not None else None, comm=comm)
        cv = ref.centerofmass(got, vel8, boxsize=None, comm=comm)
    assert cm.shape == (nlab, 3)
    d = np.abs(cm[1:] - mine["CMPosition"][1:])
    if box is not None:
        d = np.minimum(d, np.asarray(box) - d)
    assert d.max() <= 1e-12 * scale
    np.testing.assert_allclose(cv[1:], mine["CMVelocity"][1:], rtol=0, atol=1e-12 * np.abs(vel8).max())
    # the catalogue as the reference builds it (float32 columns); row 0 of the peak columns differs by design (the
    # reference pools every non-peak particle there), rows 1..H agree
    src = ref.Source({"Position": pos8, "Velocity": vel8, "Density": peak},
                     **({"BoxSize": np.asarray(box, "f8")} if box is not None else {}))
    cat = ref.fof_catalog(src, got, comm, peakcolumn="Density", periodic=box is not None)
    np.testing.assert_array_equal(cat["Length"], mine["Length"])
    for k in ("CMPosition", "PeakPosition"):
        d = np.abs(cat[k][1:] - mine[k][1:])
        if box is not None:
            d = np.minimum(d, np.asarray(box) - d)
        assert d.max() <= 1e-6 * scale, k
    for k in ("CMVelocity", "PeakVelocity"):
        np.testing.assert_allclose(cat[k][1:], mine[k][1:], rtol=1e-6, atol=1e-6 * np.abs(vel8).max())


def test_the_fixtures_cover_a_case_without_ties():
    tie_free = 0
    for name in fo.fixture_cases():
        pos, vel, peak, box, b, nmin = fo.fixture_cases()[name]
        sizes = np.bincount(fo.fof_labels(pos, b, nmin, box))[1:]
        tie_free += len(np.unique(sizes)) == len(sizes)
    assert tie_free >= 2
