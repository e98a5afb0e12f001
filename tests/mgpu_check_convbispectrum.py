"""ConvolvedFFTBispectrum on every GPU of the box (torchrun, one process per GPU) against one GPU: triangle counts
identical, B_ell and shotnoise_0 within 1e-10 of the oracle's bounds, resident and blocked.  Launched by
tests/test_gpu_convbispectrum.py::test_two_gpu_convbispectrum_matches_one_gpu."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

POLES = [0, 2, 4]


def main():
    import torch
    from nbodykit_b200 import comm as C
    from test_gpu_convbispectrum import _columns, _run, _want
    world = C.world()
    P, rank = world.size, world.rank
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    N, L, Ctr = (64, 64, 48), np.array([300., 300., 250.]), np.array([600., -200., 900.])
    cats = _columns(L, Ctr, 41, nd=4000, nr=20000)
    owner = {name: np.random.RandomState(5).randint(0, P, len(c["NZ"])) for name, c in cats.items()}
    ok = 0
    for cap in (None, 20):
        if cap:
            os.environ["NBK_BISPEC_RESIDENT"] = str(cap)
        r = _run(cats, N, L, Ctr, "f8", "tsc", True, comm=world, owner=owner, dk=0.04, poles=POLES)
        if rank == 0:
            os.environ.pop("NBK_BISPEC_RESIDENT", None)
            one = _run(cats, N, L, Ctr, "f8", "tsc", True, comm=C.SelfComm(), dk=0.04, poles=POLES)
            want = _want(one, POLES, "CompensateTSC")
            np.testing.assert_array_equal(r.poles["triangles"], one.poles["triangles"])
            a, b, c = want["rows"].T
            good = want["row_triangles"] > 0
            for ell in POLES:
                err = np.abs(r.poles["B_%d" % ell] - one.poles["B_%d" % ell])[a, b, c][good]
                assert (err <= 1e-10 * want["bound_%d" % ell][good]).all(), (cap, ell)
            i, j, l = want["triples"].T
            good = want["triangles"] > 0
            err = np.abs(r.poles["shotnoise_0"] - one.poles["shotnoise_0"])[i, j, l][good]
            assert (err <= 1e-10 * want["shot_bound"][good]).all(), cap
            ok += 1
        world.barrier()
    if rank == 0:
        print("mgpu_check_convbispectrum ok: %d GPUs, %d comparisons" % (P, ok))


if __name__ == "__main__":
    main()
