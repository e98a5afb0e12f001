"""FFTBispectrum on every GPU of the box (torchrun, one process per GPU) against one GPU: triangle counts identical and B
within 1e-12 of the oracle's bound, resident and blocked.  Launched by
tests/test_gpu_bispectrum.py::test_two_gpu_bispectrum_matches_one_gpu."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    from nbodykit_b200 import comm as C
    from oracle import bispectrum_oracle as bo
    from test_gpu_bispectrum import _field, _flat, _half, _mesh, _run
    world = C.world()
    P, rank = world.size, world.rank
    N, L = (64, 64, 48), (300., 300., 250.)
    arr = _field(N, 21)
    ok = 0
    for cap in (None, 6):
        if cap:
            os.environ["NBK_BISPEC_RESIDENT"] = str(cap)
        r = _run(_mesh(arr, L, "f8", world), dk=0.04)
        if rank == 0:
            os.environ.pop("NBK_BISPEC_RESIDENT", None)
            mesh = _mesh(arr, L, "f8", C.SelfComm())
            one = _run(mesh, dk=0.04)
            want = bo.fft_form(_half(mesh), N, L, one.bispec.edges["k1"])
            np.testing.assert_array_equal(r.bispec["triangles"], one.bispec["triangles"])
            B, _ = _flat(r, want["triples"])
            B1, _ = _flat(one, want["triples"])
            good = want["triangles"] > 0
            assert (np.abs(B - B1)[good] <= 1e-12 * want["bound"][good]).all(), cap
            ok += 1
        world.barrier()
    if rank == 0:
        print("mgpu_check_bispectrum ok: %d GPUs, %d comparisons" % (P, ok))


if __name__ == "__main__":
    main()
