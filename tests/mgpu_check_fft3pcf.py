"""FFT3PCF on every GPU of the box (torchrun, one process per GPU) against one GPU: nsep identical, corr_l within 1e-12
of the oracle's bound, resident and blocked.  Launched by tests/test_gpu_fft3pcf.py::test_two_gpu_fft3pcf_matches_one_gpu."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

POLES = [0, 1, 2, 3, 4]


def main():
    import torch
    import fft3pcf_oracle as fo
    from nbodykit_b200 import comm as C
    from test_gpu_bispectrum import _field, _mesh
    from test_gpu_fft3pcf import _corr, _run
    world = C.world()
    P, rank = world.size, world.rank
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    N, L = (64, 64, 48), (300., 300., 250.)
    F = _field(N, 42)
    e = np.linspace(0, 120., 7)
    ok = 0
    for cap in (None, 4):
        if cap:
            os.environ["NBK_BISPEC_RESIDENT"] = str(cap)
        r = _run(_mesh(F, L, "f8", world), edges=e)
        if rank == 0:
            os.environ.pop("NBK_BISPEC_RESIDENT", None)
            one = _run(_mesh(F, L, "f8", C.SelfComm()), edges=e)
            bound = fo.bound(F, N, L, e, POLES)
            np.testing.assert_array_equal(r.nsep, one.nsep)
            err = np.abs(_corr(r, POLES) - _corr(one, POLES)) / bound
            assert err.max() <= 1e-12, (cap, err.max())
            if cap:
                assert r.attrs["transforms"] > one.attrs["transforms"]
            ok += 1
        world.barrier()
    if rank == 0:
        print("mgpu_check_fft3pcf ok: %d GPUs, %d comparisons" % (P, ok))


if __name__ == "__main__":
    main()
