"""FiberCollisions on every GPU of the box (torchrun, one process per GPU) against one GPU and the oracle: Label,
Collided and NeighborID row for row on a clustered sky.

    torchrun --nproc-per-node 2 tests/mgpu_check_fibercollisions.py"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _np(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def main():
    from nbodykit_b200 import comm as C
    from nbodykit_b200.lab import FiberCollisions
    from oracle import fibercollisions_oracle as fo
    world = C.world()
    P, rank = world.size, world.rank
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    rng = np.random.RandomState(31)
    ra, dec = rng.uniform(100, 105, 80000), rng.uniform(-2.5, 2.5, 80000)
    c = rng.uniform([100, -2.5], [105, 2.5], size=(30, 2))
    k = rng.randint(0, 30, 20000)
    ra = np.concatenate([ra, c[k, 0] + rng.normal(scale=0.03, size=20000)])
    dec = np.concatenate([dec, c[k, 1] + rng.normal(scale=0.03, size=20000)])
    n = len(ra)
    mine = slice(rank * n // P, (rank + 1) * n // P)
    r = FiberCollisions(ra[mine], dec[mine], seed=17, comm=world)
    cols = [np.concatenate(world.allgather(_np(r.labels[c].compute()))) for c in ('Label', 'Collided', 'NeighborID')]
    if rank == 0:
        one = FiberCollisions(ra, dec, seed=17, comm=C.SelfComm())
        want = [_np(one.labels[c].compute()) for c in ('Label', 'Collided', 'NeighborID')]
        assert all(np.array_equal(a, b) for a, b in zip(cols, want)), "differs from one GPU"
        pos = one.source['Position'].compute().cpu().numpy()
        o = fo.fiber_collisions(pos, one._collision_radius_rad, 17)
        assert all(np.array_equal(a, b) for a, b in zip(want, o)), "differs from the oracle"
        print("mgpu_check_fibercollisions ok: %d GPUs, %d rows, %d collided, largest group %d"
              % (P, n, int(cols[1].sum()), one._stats['largest']))
    world.barrier()


if __name__ == "__main__":
    main()
