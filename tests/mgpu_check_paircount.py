"""Pair counts on every GPU of the box (torchrun, one process per GPU) against one GPU: npairs identical in every mode,
periodic and not, auto and cross.  Launched by tests/test_gpu_paircount.py::test_two_gpu_paircount_matches_one_gpu."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    from nbodykit_b200 import comm as C
    from nbodykit_b200.lab import ArrayCatalog, SimulationBoxPairCount
    world = C.world()
    P, rank = world.size, world.rank
    rng = np.random.RandomState(41)
    L = 100.
    a = (rng.uniform(size=(60000, 3)) * L).astype("f4")
    b = rng.uniform(size=(30000, 3)) * L
    w = rng.uniform(0.5, 2., len(a))
    edges = np.linspace(1., 20., 9)

    def cat(pos, wt, comm, mine=True):
        n = len(pos)
        sl = slice(rank * n // P, (rank + 1) * n // P) if mine else slice(0, n)
        data = {"Position": torch.from_numpy(np.ascontiguousarray(pos[sl])).cuda()}
        if wt is not None:
            data["Weight"] = torch.from_numpy(np.ascontiguousarray(wt[sl])).cuda()
        return ArrayCatalog(data, comm=comm, BoxSize=[L] * 3)
    ok = 0
    for mode, kw in (("1d", {}), ("2d", dict(Nmu=8)), ("projected", dict(pimax=15.))):
        for periodic in (True, False):
            for cross in (False, True):
                second = cat(b, None, world) if cross else None
                r = SimulationBoxPairCount(mode, cat(a, w, world), edges, periodic=periodic, second=second, **kw)
                if rank == 0:
                    one = SimulationBoxPairCount(mode, cat(a, w, one_comm(), False), edges, periodic=periodic,
                                                 second=cat(b, None, one_comm(), False) if cross else None, **kw)
                    assert np.array_equal(r.pairs["npairs"], one.pairs["npairs"]), (mode, periodic, cross)
                    np.testing.assert_allclose(r.pairs["wnpairs"], one.pairs["wnpairs"], rtol=1e-12)
                    ok += 1
    if rank == 0:
        print("mgpu_check_paircount ok: %d GPUs, %d comparisons" % (P, ok))
    world.barrier()


_ONE = []


def one_comm():
    from nbodykit_b200 import comm as C
    if not _ONE:
        _ONE.append(C.SelfComm())
    return _ONE[0]


if __name__ == "__main__":
    main()
