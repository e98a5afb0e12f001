"""Survey pair counts on every GPU of the box (torchrun, one process per GPU) against one GPU: npairs identical in every
mode, auto and cross.  Launched by tests/test_gpu_survey_paircount.py::test_two_gpu_survey_matches_one_gpu."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    from nbodykit_b200 import comm as C
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200.lab import ArrayCatalog, SurveyDataPairCount
    from oracle.survey_paircount_oracle import sky_catalogue
    world = C.world()
    P, rank = world.size, world.rank
    a = sky_catalogue(41, 40000)
    b = sky_catalogue(42, 20000)
    w = np.random.RandomState(43).uniform(0.5, 2., len(a[0]))

    def cat(s, wt, comm, mine=True):
        n = len(s[0])
        sl = slice(rank * n // P, (rank + 1) * n // P) if mine else slice(0, n)
        data = {k: torch.from_numpy(np.ascontiguousarray(v[sl])).cuda() for k, v in zip(("RA", "DEC", "Redshift"), s)}
        if wt is not None:
            data["Weight"] = torch.from_numpy(np.ascontiguousarray(wt[sl])).cuda()
        return ArrayCatalog(data, comm=comm)
    ok = 0
    for mode, edges, kw in (("1d", np.linspace(10., 80., 8), {}), ("2d", np.linspace(10., 80., 8), dict(Nmu=8)),
                            ("projected", np.linspace(10., 80., 8), dict(pimax=40.)),
                            ("angular", np.logspace(-1, 0.5, 7), {})):
        for cross in (False, True):
            second = cat(b, None, world) if cross else None
            r = SurveyDataPairCount(mode, cat(a, w, world), edges, cosmo=Planck15, second=second, **kw)
            if rank == 0:
                one = SurveyDataPairCount(mode, cat(a, w, one_comm(), False), edges, cosmo=Planck15,
                                          second=cat(b, None, one_comm(), False) if cross else None, **kw)
                assert np.array_equal(r.pairs["npairs"], one.pairs["npairs"]), (mode, cross)
                np.testing.assert_allclose(r.pairs["wnpairs"], one.pairs["wnpairs"], rtol=1e-12)
                ok += 1
    if rank == 0:
        print("mgpu_check_survey ok: %d GPUs, %d comparisons" % (P, ok))
    world.barrier()


_ONE = []


def one_comm():
    from nbodykit_b200 import comm as C
    if not _ONE:
        _ONE.append(C.SelfComm())
    return _ONE[0]


if __name__ == "__main__":
    main()
