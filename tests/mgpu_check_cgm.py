"""CylindricalGroups on every GPU of the box (torchrun, one process per GPU) against one GPU and the float64 oracle: all
three columns row for row, for a flat-sky periodic box and an observer at the origin.

    torchrun --nproc-per-node 2 tests/mgpu_check_cgm.py"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

COLS = ("cgm_type", "cgm_haloid", "num_cgm_sats")


def main():
    from nbodykit_b200 import comm as C
    from nbodykit_b200.lab import ArrayCatalog, CylindricalGroups
    from oracle import cgm_oracle as co
    world = C.world()
    P, rank = world.size, world.rank
    rng = np.random.RandomState(31)
    L = 64.
    pos = rng.uniform(size=(40000, 3)) * L
    centres = rng.uniform(size=(40, 3)) * L
    pos = np.concatenate([pos, (centres[rng.randint(0, 40, 20000)] + rng.normal(scale=0.8, size=(20000, 3))) % L])
    m = rng.uniform(size=len(pos))
    n = len(pos)
    mine = slice(rank * n // P, (rank + 1) * n // P)
    for los, periodic, shift in (([0, 0, 1], True, 0.), (None, False, 100.)):
        p = pos + shift
        cat = ArrayCatalog({"Position": torch.from_numpy(p[mine]).cuda(), "m": torch.from_numpy(m[mine]).cuda()},
                           comm=world, BoxSize=[L] * 3)
        r = CylindricalGroups(cat, "m", 1.0, 2.0, flat_sky_los=los, periodic=periodic)
        got = {c: np.concatenate(world.allgather(np.asarray(r.groups[c].compute()))) for c in COLS}
        if rank == 0:
            one = CylindricalGroups(ArrayCatalog({"Position": torch.from_numpy(p).cuda(), "m": torch.from_numpy(m).cuda()},
                                                 comm=C.SelfComm(), BoxSize=[L] * 3), "m", 1.0, 2.0, flat_sky_los=los,
                                    periodic=periodic)
            want = co.cgm(p, [m], 1.0, 2.0, los=los, periodic=periodic, BoxSize=L)
            for k, c in enumerate(COLS):
                assert np.array_equal(got[c], np.asarray(one.groups[c].compute())), "%s differs from one GPU" % c
                assert np.array_equal(got[c], want[k]), "%s differs from the oracle" % c
            print("mgpu_check_cgm ok: %d GPUs, %d rows, los %s, %d satellites, %d rounds"
                  % (P, n, los, int(got["cgm_type"].sum()), r.rounds))
        world.barrier()


if __name__ == "__main__":
    main()
