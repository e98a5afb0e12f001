"""The three-point function on every GPU of the box (torchrun, one process per GPU) against one GPU: npairs identical
and zeta within 1e-12 of the oracle's bound B, periodic and not.  Launched by
tests/test_gpu_threeptcf.py::test_two_gpu_threeptcf_matches_one_gpu."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    from nbodykit_b200 import comm as C
    from nbodykit_b200.lab import ArrayCatalog, SimulationBox3PCF
    from oracle import threeptcf_oracle as to
    world = C.world()
    P, rank = world.size, world.rank
    rng = np.random.RandomState(43)
    L = 60.
    a = (rng.uniform(size=(20000, 3)) * L).astype("f4")
    w = rng.uniform(-0.5, 2., len(a))
    edges, poles = np.linspace(0., 5., 6), [0, 1, 2, 3]

    def cat(comm, mine=True):
        n = len(a)
        sl = slice(rank * n // P, (rank + 1) * n // P) if mine else slice(0, n)
        data = {"Position": torch.from_numpy(np.ascontiguousarray(a[sl])).cuda(),
                "Weight": torch.from_numpy(np.ascontiguousarray(w[sl])).cuda()}
        return ArrayCatalog(data, comm=comm, BoxSize=[L] * 3)
    ok = 0
    for periodic in (True, False):
        r = SimulationBox3PCF(cat(world), poles, edges, periodic=periodic)
        if rank == 0:
            one = SimulationBox3PCF(cat(one_comm(), False), poles, edges, periodic=periodic)
            assert np.array_equal(r.npairs, one.npairs), periodic
            bound = to.compute(a, edges, poles, box=[L] * 3 if periodic else None, w=w)["bound"]
            for i, ell in enumerate(poles):
                err = np.abs(r.poles["corr_%d" % ell] - one.poles["corr_%d" % ell])
                assert (err <= 1e-12 * bound[i]).all(), (periodic, ell)
            ok += 1
    if rank == 0:
        print("mgpu_check_threeptcf ok: %d GPUs, %d comparisons" % (P, ok))
    world.barrier()


_ONE = []


def one_comm():
    from nbodykit_b200 import comm as C
    if not _ONE:
        _ONE.append(C.SelfComm())
    return _ONE[0]


if __name__ == "__main__":
    main()
