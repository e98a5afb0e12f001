"""
Writes tests/golden/fof_*.npz from the REFERENCE's own FOF helpers (nbodykit/algorithms/fof.py, loaded verbatim by
oracle/fof_refload.py): for each catalogue of oracle.fof_oracle.fixture_cases(), the groups of the float64 kd-tree
partition are labelled by the reference's `_assign_labels`, and `fof_catalog` computes the features from those labels.
The GPU machines have no reference tree, so the outputs are committed.  Re-run: `python tests/golden/make_fof_golden.py`.

Stored: inputs (pos, vel, peak, box (NaN when non-periodic), b, nmin), `labels` of the reference, `ties` (whether two
groups of label > 0 have the same size, where the reference's order is not reproducible), and the reference catalogue
columns Length, CMPosition, CMVelocity, PeakPosition, PeakVelocity (float32 as the reference stores them).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import fof_oracle as fo, fof_refload  # noqa: E402


def main():
    ref = fof_refload.load()
    comm = ref.Comm()
    for name, (pos, vel, peak, box, b, nmin) in fo.fixture_cases().items():
        mid = fo.minid(pos, b, box)
        labels = np.asarray(ref._assign_labels(mid, comm=comm, thresh=nmin))
        sizes = np.bincount(labels)[1:]
        src = ref.Source({"Position": pos, "Velocity": vel, "Density": peak},
                         **({"BoxSize": np.asarray(box, "f8")} if box is not None else {}))
        cat = ref.fof_catalog(src, labels, comm, peakcolumn="Density", periodic=box is not None)
        np.savez_compressed(os.path.join(HERE, "fof_%s.npz" % name), pos=pos, vel=vel, peak=peak,
                            box=np.asarray(box if box is not None else [np.nan] * 3, "f8"), b=b, nmin=nmin,
                            labels=labels, ties=len(np.unique(sizes)) != len(sizes),
                            **{k: cat[k] for k in cat.dtype.names})
        print(name, len(pos), "particles", len(sizes), "groups", "ties" if len(np.unique(sizes)) != len(sizes) else "")


if __name__ == "__main__":
    main()
