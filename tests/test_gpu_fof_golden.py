"""FOF on the GPU against the fixtures the reference's own helpers produced (tests/golden/fof_*.npz, written by
tests/golden/make_fof_golden.py from nbodykit/algorithms/fof.py's `_assign_labels` and `fof_catalog`): identical labels
where no two groups share a size (the reference orders ties with an unstable sort), else the same partition and sizes;
features of rows 1..H to 2e-6 of the box (float32 columns)."""
import glob
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "fof_*.npz")))


def test_fixtures_present():
    assert len(FIXTURES) >= 4


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p)[4:-4] for p in FIXTURES])
def test_labels_and_features_equal_the_reference(cuda, path):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ArrayCatalog, FOF
    z = np.load(path)
    periodic = not np.isnan(z["box"]).any()
    box = z["box"] if periodic else None
    cols = {k: torch.as_tensor(z[c]).cuda() for k, c in (("Position", "pos"), ("Velocity", "vel"), ("Density", "peak"))}
    cat = ArrayCatalog(cols, comm=SelfComm(), **({"BoxSize": box} if periodic else {}))
    fof = FOF(cat, linking_length=float(z["b"]), nmin=int(z["nmin"]), absolute=True, periodic=periodic)
    want = z["labels"]
    if bool(z["ties"]):
        pairs = set(zip(fof.labels.tolist(), want.tolist()))
        assert len(pairs) == len(set(want.tolist())) == len(set(fof.labels.tolist()))
        assert sorted(np.bincount(fof.labels)[1:]) == sorted(np.bincount(want)[1:])
        return
    np.testing.assert_array_equal(fof.labels, want)
    feat = fof.find_features(peakcolumn="Density")
    np.testing.assert_array_equal(np.asarray(feat["Length"]), z["Length"])
    scale = float(np.max(box)) if periodic else float(np.ptp(z["pos"]))
    for k in ("CMPosition", "PeakPosition"):
        d = np.abs(np.asarray(feat[k])[1:].astype("f8") - z[k][1:])
        if periodic:
            d = np.minimum(d, box - d)
        assert d.max() <= 2e-6 * scale, k
    vmax = np.abs(z["vel"]).max()
    for k in ("CMVelocity", "PeakVelocity"):
        np.testing.assert_allclose(np.asarray(feat[k])[1:], z[k][1:], rtol=2e-6, atol=2e-6 * vmax)
