"""KDDensity on every GPU of the box (torchrun, one process per GPU) against one GPU and the oracle: the distance and
the density row for row, for a clustered float32 catalogue at several margins.

    torchrun --nproc-per-node 2 tests/mgpu_check_kddensity.py"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    from nbodykit_b200 import comm as C
    from nbodykit_b200.lab import ArrayCatalog, KDDensity
    from oracle import kddensity_oracle as ko
    world = C.world()
    P, rank = world.size, world.rank
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    rng = np.random.RandomState(31)
    L = 64.
    pos = rng.uniform(size=(40000, 3)) * L
    centres = rng.uniform(size=(40, 3)) * L
    pos = np.concatenate([pos, (centres[rng.randint(0, 40, 20000)] + rng.normal(scale=0.8, size=(20000, 3))) % L])
    pos = pos.astype("f4")
    n = len(pos)
    mine = slice(rank * n // P, (rank + 1) * n // P)
    for margin in (0.0, 1.0, 8.0):
        cat = ArrayCatalog({"Position": torch.from_numpy(pos[mine]).cuda()}, comm=world, BoxSize=L)
        r = KDDensity(cat, margin=margin)
        d = np.concatenate(world.allgather(r._distance))
        dens = np.concatenate(world.allgather(r.density))
        phase2 = int(world.allreduce(r._stats["phase2_rows"]))
        if rank == 0:
            one = KDDensity(ArrayCatalog({"Position": torch.from_numpy(pos).cuda()}, comm=C.SelfComm(), BoxSize=L))
            want_d, want = ko.density(pos, L)
            assert np.array_equal(d, one._distance) and np.array_equal(dens, one.density), "differs from one GPU"
            assert np.array_equal(d, want_d), "distance differs from the oracle"
            np.testing.assert_allclose(dens, want, rtol=1e-15, atol=0)
            print("mgpu_check_kddensity ok: %d GPUs, %d rows, margin %g, %d rows in phase 2" % (P, n, margin, phase2))
        world.barrier()


if __name__ == "__main__":
    main()
