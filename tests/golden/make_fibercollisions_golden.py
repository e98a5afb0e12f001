"""
Regenerate tests/golden/fibercollisions_*.npz: ra, dec, seed, collision radius and the reference's own Label, Collided
and NeighborID (nbodykit/algorithms/fibercollisions.py, run verbatim on one rank by oracle/fibercollisions_refload.py),
checked here against the restatement of oracle/fibercollisions_oracle.py with NumPy's global generator as chooser and the
reference's member order.  `forced` marks the rows of groups whose greedy never had more than one candidate: there the
result does not depend on the random choices.  Needs the reference tree; the fixtures let GPU machines compare against
the reference without it.

    python tests/golden/make_fibercollisions_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import fibercollisions_oracle as fo, fibercollisions_refload as fr  # noqa: E402

RAD62 = 62 / 60. / 60.


def cases():
    """name -> (ra, dec, collision radius in degrees, seed)"""
    out = {}
    # the reference test's catalogue: 10^4 rows in 10 x 5 degrees
    np.random.seed(42)
    ra = 10. * np.random.random(size=10000)
    dec = 5. * np.random.random(size=10000) - 5.0
    out["reference"] = (ra, dec, RAD62, 42)
    # 4000 per square degree over 1.6 x 1.6 degrees: groups of hundreds of members
    rng = np.random.RandomState(7)
    n = int(4000 * 1.6 * 1.6)
    ra = 30 + 1.6 * rng.random_sample(n)
    dec = np.rad2deg(np.arcsin(rng.uniform(np.sin(np.deg2rad(10)), np.sin(np.deg2rad(11.6)), n)))
    out["dense"] = (ra, dec, RAD62, 3)
    out["issue584_3pt"] = (np.array([0., 1., 2.]), np.array([0., 0., 0.]), 1.5, 0)
    out["issue584_4pt"] = (np.array([0., 1., 2., 10.]), np.array([0., 0., 0., 0.]), 1.5, 0)
    return out


def _check_margin(pos, label, rad):
    """no pair lies within 1e-9 rad^2 of the FOF threshold (float64) or within 1e-9 rad of the collision radius
    (float32 positions), so that an ulp of the sky transform cannot change the answer"""
    from oracle import fof_oracle
    fof_oracle.friend_pairs(pos, rad, [fo.BOX] * 3, check_margin=True)
    p4 = pos.astype("f4")
    for lab in np.unique(label[label > 0]):
        mem = np.nonzero(label == lab)[0]
        d = fo._dist(p4[mem][:, None, :], p4[mem][None, :, :])
        assert not np.any(np.abs(d - rad) < 1e-9 * rad), "a member separation is too close to the collision radius"


def main():
    for name, (ra, dec, crad, seed) in cases().items():
        pos, lab, col, nb, rad = fr.run(ra, dec, collision_radius=crad, seed=seed)
        _check_margin(pos, lab, rad)
        state = np.random.get_state()
        np.random.seed(seed)
        c2, n2, forced = fo.assign(pos, lab, rad, fo.numpy_chooser(), order="reference", full=True)
        np.random.set_state(state)
        assert np.array_equal(col, c2) and np.array_equal(nb, n2), name
        assert np.array_equal(lab, fo.fof_labels(fo.unit_sphere(ra, dec), rad)), name
        np.savez_compressed(os.path.join(HERE, "fibercollisions_%s.npz" % name), ra=ra, dec=dec,
                            collision_radius=np.float64(crad), seed=np.int64(seed), Label=lab.astype("i4"),
                            Collided=col.astype("i1"), NeighborID=nb.astype("i4"), forced=forced)
        sizes = np.bincount(lab)[1:]
        print(name, len(ra), "rows,", len(sizes), "groups, largest", sizes.max() if len(sizes) else 0, ",",
              int(col.sum()), "collided,", int(forced[lab > 0].sum()), "grouped rows forced")


if __name__ == "__main__":
    main()
