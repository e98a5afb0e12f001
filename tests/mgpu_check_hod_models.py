"""HaloCatalog.populate with Hearin15Model and Leauthaud11Model on every GPU of the box (torchrun, one process per GPU)
against one GPU and the oracle: the galaxies of all ranks, sorted by (gal_type, halo_id, satellite), equal the one-GPU
catalogue column for column (for Hearin15 this needs the percentiles ranked over all ranks), and the one-GPU catalogue
equals the float64 oracle's rows.

    torchrun --nproc-per-node 2 tests/mgpu_check_hod_models.py"""
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
    from nbodykit_b200.lab import Hearin15Model, Leauthaud11Model
    from test_gpu_hod import assert_matches, host_cols, make_halos
    from test_gpu_hod_models import halo_catalog, oracle_for
    world = C.world()
    P, rank = world.size, world.rank
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    mass, pos, vel = make_halos(300000, 21, 1000., hi=14.8)
    n = mass.size
    mine = slice(rank * n // P, (rank + 1) * n // P)
    for model in (Hearin15Model(split=0.4, mean_occupation_satellites_assembias_param1=-0.5), Leauthaud11Model()):
        cat = halo_catalog(mass[mine], pos[mine], vel[mine], 1000., 0.55, comm=world).populate(model, seed=31)
        parts = world.allgather(host_cols(cat))
        if rank == 0:
            one = halo_catalog(mass, pos, vel, 1000., 0.55, comm=SelfComm())
            want = host_cols(one.populate(model, seed=31))
            cols = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
            order = np.lexsort((cols["halo_id"], cols["gal_type"]))
            for k in want:
                np.testing.assert_array_equal(cols[k][order], want[k], err_msg=k)
            assert_matches(want, oracle_for(one, model, 31), np.full(3, 1000.))
            print("mgpu_check_hod_models ok: %s, %d ranks, %d galaxies equal one GPU and the oracle"
                  % (type(model).__name__, P, len(order)))


if __name__ == "__main__":
    main()
