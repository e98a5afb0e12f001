"""FOF on every GPU of the box (torchrun, one process per GPU) against one GPU: labels and the gathered feature catalogue.
Launched by tests/test_gpu_fof.py::test_two_gpu_fof_matches_one_gpu."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    from nbodykit_b200 import comm as C
    from nbodykit_b200.lab import ArrayCatalog, FOF
    world = C.world()
    P, rank = world.size, world.rank
    rng = np.random.RandomState(31)
    L = 64.
    pos = (rng.uniform(size=(40000, 3)) * L).astype("f4")
    centres = rng.uniform(size=(40, 3)) * L
    clump = ((centres[rng.randint(0, 40, 20000)] + rng.normal(scale=0.4, size=(20000, 3))) % L).astype("f4")
    pos = np.concatenate([pos, clump])
    pos = pos[np.argsort(pos[:, 0], kind="stable")]
    vel = rng.normal(size=pos.shape).astype("f4")
    n = len(pos)
    mine = slice(rank * n // P, (rank + 1) * n // P)
    cat = ArrayCatalog({"Position": torch.from_numpy(pos[mine]).cuda(), "Velocity": torch.from_numpy(vel[mine]).cuda()},
                       comm=world, BoxSize=[L] * 3)
    fof = FOF(cat, linking_length=0.5, nmin=5, absolute=True)
    feat = fof.find_features()
    labels = np.concatenate(world.allgather(fof.labels))
    length = np.concatenate(world.allgather(np.asarray(feat["Length"])))
    cm = np.concatenate(world.allgather(np.asarray(feat["CMPosition"])))
    if rank == 0:
        one = FOF(ArrayCatalog({"Position": torch.from_numpy(pos).cuda(), "Velocity": torch.from_numpy(vel).cuda()},
                               comm=C.SelfComm(), BoxSize=[L] * 3), linking_length=0.5, nmin=5, absolute=True)
        f1 = one.find_features()
        assert np.array_equal(labels, one.labels), "labels differ from one GPU"
        assert np.array_equal(length, np.asarray(f1["Length"])), "group sizes differ from one GPU"
        np.testing.assert_allclose(cm[1:], np.asarray(f1["CMPosition"])[1:], rtol=1e-6, atol=1e-6 * L)
        print("mgpu_check_fof ok: %d GPUs, %d particles, %d groups, %d merge rounds" % (P, n, labels.max(), fof.merge_rounds))
    world.barrier()


if __name__ == "__main__":
    main()
