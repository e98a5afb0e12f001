"""FiberCollisions without a GPU: argument errors (raised before any device work), the hashed chooser shared by the
package and the oracle, and the invariants of the oracle's answer."""
import numpy as np
import pytest

from oracle import fibercollisions_oracle as fo


def _fc(**kw):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import FiberCollisions
    return FiberCollisions(comm=SelfComm(), **kw)


@pytest.mark.parametrize("kw,msg", [
    (dict(ra=[1., 2.], dec=[1.]), "different lengths"),
    (dict(ra=[np.nan, 1.], dec=[1., 2.]), "must be finite"),
    (dict(ra=[1., 2.], dec=[np.inf, 2.]), "must be finite"),
    (dict(ra=np.ones((2, 2)), dec=np.ones((2, 2))), "one-dimensional"),
    (dict(ra=[1.], dec=[1.], collision_radius=0.), "collision_radius must be positive"),
    (dict(ra=[1.], dec=[1.], collision_radius=-1.), "collision_radius must be positive"),
    (dict(ra=[1.], dec=[1.], collision_radius=np.inf), "collision_radius must be positive"),
    (dict(ra=[1.], dec=[1.], seed=-1), "seed must be an integer"),
    (dict(ra=[1.], dec=[1.], seed=2 ** 32), "seed must be an integer"),
    (dict(ra=[1.], dec=[1.], seed=1.5), "seed must be an integer"),
    (dict(ra=[1.], dec=[1.], collision_radius=1e-5), "below the smallest"),
])
def test_argument_errors(kw, msg):
    with pytest.raises(ValueError, match=msg):
        _fc(**kw)


def test_hash_is_shared_and_reproducible():
    from nbodykit_b200.algorithms.fibercollisions import hash_pick
    choose = fo.hash_chooser(12345)
    rng = np.random.RandomState(0)
    for g, step, k in zip(rng.randint(0, 2 ** 31, 200), rng.randint(0, 10 ** 6, 200), rng.randint(1, 5000, 200)):
        p = hash_pick(12345, g, step, k)
        assert 0 <= p < k and p == choose(g, step, k) == hash_pick(12345, g, step, k)
    # SplitMix64 of 0 is its published first output
    assert fo._splitmix(0) == 0xE220A8397B1DCDAF
    # the picks of one group change with the seed and the step
    assert len({hash_pick(s, 7, 0, 1000) for s in range(20)}) > 15
    assert len({hash_pick(1, 7, t, 1000) for t in range(20)}) > 15


@pytest.mark.parametrize("seed", [0, 1, 99])
def test_oracle_invariants(seed):
    rng = np.random.RandomState(seed)
    n = 12000
    ra = rng.uniform(20, 22, n)
    dec = np.rad2deg(np.arcsin(rng.uniform(np.sin(np.deg2rad(-1.)), np.sin(np.deg2rad(0.5)), n)))
    pos = fo.unit_sphere(ra, dec)
    rad = np.deg2rad(62 / 3600.)
    lab, col, nb = fo.fiber_collisions(pos, rad, seed)
    assert np.bincount(lab)[1:].max() > 32
    fo.check_invariants(pos, lab, col, nb, rad)
    # stopping at the first removal without a collider gives the answer of the full loop
    c2, n2, _ = fo.assign(pos, lab, rad, fo.hash_chooser(seed), full=True)
    np.testing.assert_array_equal(col, c2)
    np.testing.assert_array_equal(nb, n2)
