"""The restatement of oracle/fibercollisions_oracle.py reproduces the reference's FiberCollisions (run verbatim on one
rank by oracle/fibercollisions_refload.py) exactly when it draws from NumPy's global generator and orders the members as
the reference does: on the reference test's catalogue at several seeds, a dense field with groups of hundreds of members
and the issue-584 rows.  Skips without the reference tree."""
import numpy as np
import pytest

from oracle import fibercollisions_oracle as fo
from oracle import fibercollisions_refload as fr

pytestmark = pytest.mark.skipif(not fr.available(), reason="reference tree not present")


def _compare(ra, dec, seed, collision_radius=62 / 3600.):
    pos, lab, col, nb, rad = fr.run(ra, dec, collision_radius=collision_radius, seed=seed)
    np.testing.assert_array_equal(lab, fo.fof_labels(fo.unit_sphere(ra, dec), rad))
    state = np.random.get_state()
    try:
        np.random.seed(seed)
        c2, n2, forced = fo.assign(pos, lab, rad, fo.numpy_chooser(), order="reference", full=True)
    finally:
        np.random.set_state(state)
    np.testing.assert_array_equal(col, c2)
    np.testing.assert_array_equal(nb, n2)
    return lab, col, nb


@pytest.mark.parametrize("seed", [0, 3, 42])
def test_reference_catalogue(seed):
    np.random.seed(42)
    ra = 10. * np.random.random(size=10000)
    dec = 5. * np.random.random(size=10000) - 5.0
    lab, col, nb = _compare(ra, dec, seed)
    assert col.sum() == 817 and lab.max() == 773


def test_dense_field():
    rng = np.random.RandomState(8)
    n = int(4000 * 1.2 * 1.2)
    ra = 50 + 1.2 * rng.random_sample(n)
    dec = np.rad2deg(np.arcsin(rng.uniform(np.sin(np.deg2rad(-20)), np.sin(np.deg2rad(-18.8)), n)))
    lab, col, nb = _compare(ra, dec, 5)
    assert np.bincount(lab)[1:].max() > 32


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_issue584(seed):
    _, col, nb = _compare(np.array([0., 1., 2.]), np.zeros(3), seed, 1.5)
    assert list(col) == [0, 1, 0] and list(nb) == [-1, 0, -1]
    _, col, nb = _compare(np.array([0., 1., 2., 10.]), np.zeros(4), seed, 1.5)
    assert list(col) == [0, 1, 0, 0] and list(nb) == [-1, 0, -1, -1]
