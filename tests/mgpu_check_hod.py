"""HaloCatalog.populate on every GPU of the box (torchrun, one process per GPU) against one GPU and the oracle: the
galaxies of all ranks, sorted by (gal_type, halo_id, satellite), equal the one-GPU catalogue column for column, and the
one-GPU catalogue equals the float64 oracle's rows.

    torchrun --nproc-per-node 2 tests/mgpu_check_hod.py"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    from nbodykit_b200 import comm as C
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import Zheng07Model
    from test_gpu_hod import DEFAULTS, assert_matches, halo_catalog, host_cols, make_halos, oracle_for
    world = C.world()
    P, rank = world.size, world.rank
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    mass, pos, vel = make_halos(300000, 21, 1000.)
    n = mass.size
    mine = slice(rank * n // P, (rank + 1) * n // P)
    cat = halo_catalog(mass[mine], pos[mine], vel[mine], 1000., comm=world).populate(Zheng07Model, seed=31)
    parts = world.allgather(host_cols(cat))
    if rank == 0:
        one = halo_catalog(mass, pos, vel, 1000., comm=SelfComm())
        want = host_cols(one.populate(Zheng07Model, seed=31))
        cols = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
        order = np.lexsort((cols["halo_id"], cols["gal_type"]))
        for k in want:
            np.testing.assert_array_equal(cols[k][order], want[k], err_msg=k)
        assert_matches(want, oracle_for(one, DEFAULTS, 31), np.full(3, 1000.))
        print("mgpu_check_hod ok: %d ranks, %d galaxies equal one GPU and the oracle" % (P, len(order)))


if __name__ == "__main__":
    main()
