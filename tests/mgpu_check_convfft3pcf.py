"""ConvolvedFFT3PCF on every GPU of the box (torchrun, one process per GPU) against one GPU: nsep identical, nnn_l and
rrr_l within 1e-12 of the oracle's bounds, resident and blocked.  Launched by
tests/test_gpu_convfft3pcf.py::test_two_gpu_convfft3pcf_matches_one_gpu."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    import torch
    import convfft3pcf_oracle as cfo
    from nbodykit_b200 import comm as C
    from test_gpu_convfft3pcf import _columns, _fields, _run, _stack
    world = C.world()
    P, rank = world.size, world.rank
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    N, L, Ctr = (64, 64, 48), np.array([300., 300., 250.]), np.array([600., -200., 900.])
    e = np.linspace(0, 50., 5)
    cats = _columns(Ctr, 80., 41, nd=4000, nr=20000)
    owner = {name: np.random.RandomState(5).randint(0, P, len(c["NZ"])) for name, c in cats.items()}
    ok = 0
    for cap in (None, 3):
        if cap:
            os.environ["NBK_BISPEC_RESIDENT"] = str(cap)
        r = _run(cats, N, L, Ctr, "f8", "tsc", True, comm=world, owner=owner, edges=e)
        if rank == 0:
            os.environ.pop("NBK_BISPEC_RESIDENT", None)
            one = _run(cats, N, L, Ctr, "f8", "tsc", True, comm=C.SelfComm(), edges=e)
            Nf, Rf = _fields(one)
            want = cfo.fft_form(Nf, Rf, N, L, e, [0, 1, 2, 3, 4])
            np.testing.assert_array_equal(r.nsep, one.nsep)
            for kind, bk in (("nnn", "bound_n"), ("rrr", "bound_r")):
                err = np.abs(_stack(r, kind) - _stack(one, kind)) / want[bk]
                assert err.max() <= 1e-12, (cap, kind, err.max())
            if cap:
                assert r.attrs["transforms"] > one.attrs["transforms"]
            ok += 1
        world.barrier()
    if rank == 0:
        print("mgpu_check_convfft3pcf ok: %d GPUs, %d comparisons" % (P, ok))


if __name__ == "__main__":
    main()
