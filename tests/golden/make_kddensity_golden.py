"""
Regenerate tests/golden/kddensity_*.npz: positions, BoxSize and the density of the reference's own KDDensity
(nbodykit/algorithms/kdtree.py, run verbatim on one rank by oracle/kddensity_refload.py), checked here against the
restatement of oracle/kddensity_oracle.py.  Needs the reference tree; the fixtures let GPU machines compare against the
reference without it.

    python tests/golden/make_kddensity_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import kddensity_oracle as ko, kddensity_refload as kr  # noqa: E402


def cases():
    """name -> (pos, BoxSize): uniform float32 rows, and float64 clumps with coincident rows over a background"""
    out = {}
    rng = np.random.RandomState(42)
    L = 64.
    out["uniform_f4"] = ((rng.uniform(size=(1500, 3)) * L).astype("f4"), L)
    centres = rng.uniform(size=(12, 3)) * L
    clumps = (centres[rng.randint(0, 12, 900)] + rng.normal(scale=0.7, size=(900, 3))) % L
    dup = np.repeat(clumps[:3], 9, axis=0)
    out["clustered_f8"] = (np.concatenate([rng.uniform(size=(400, 3)) * L, clumps, dup]), L)
    return out


def main():
    for name, (pos, L) in cases().items():
        dens, _ = kr.run(pos, L)
        _, mine = ko.density(pos, L)
        assert np.array_equal(dens, mine), name
        np.savez_compressed(os.path.join(HERE, "kddensity_%s.npz" % name), pos=pos, BoxSize=np.float64(L), density=dens)
        print(name, len(pos), "rows,", int(np.isinf(dens).sum()), "infinite")


if __name__ == "__main__":
    main()
