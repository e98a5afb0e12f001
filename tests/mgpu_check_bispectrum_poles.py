"""FFTBispectrum multipoles on every GPU of the box (torchrun, one process per GPU) against one GPU: triangle counts
identical and B_ell within 1e-12 of the oracle's bound, resident and blocked.  Launched by
tests/test_gpu_bispectrum_poles.py::test_two_gpu_bispectrum_poles_matches_one_gpu."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

POLES = [0, 2, 4]
LOS = list(np.ones(3) / np.sqrt(3))


def main():
    from nbodykit_b200 import comm as C
    import bispectrum_poles_oracle as bpo
    from test_gpu_bispectrum import _field, _half, _mesh, _run
    world = C.world()
    P, rank = world.size, world.rank
    N, L = (64, 64, 48), (300., 300., 250.)
    arr = _field(N, 21)
    ok = 0
    for cap in (None, 20):
        if cap:
            os.environ["NBK_BISPEC_RESIDENT"] = str(cap)
        r = _run(_mesh(arr, L, "f8", world), dk=0.04, poles=POLES, los=LOS)
        if rank == 0:
            os.environ.pop("NBK_BISPEC_RESIDENT", None)
            mesh = _mesh(arr, L, "f8", C.SelfComm())
            one = _run(mesh, dk=0.04, poles=POLES, los=LOS)
            want = bpo.fft_form_poles(_half(mesh), N, L, one.bispec.edges["k1"], POLES, LOS)
            np.testing.assert_array_equal(r.poles["triangles"], one.poles["triangles"])
            for ell in POLES:
                a, b, c = want[ell]["rows"].T
                good = want[ell]["triangles"] > 0
                err = np.abs(r.poles["B_%d" % ell][a, b, c] - one.poles["B_%d" % ell][a, b, c])[good]
                assert (err <= 1e-12 * want[ell]["bound"][good]).all(), (cap, ell)
            ok += 1
        world.barrier()
    if rank == 0:
        print("mgpu_check_bispectrum_poles ok: %d GPUs, %d comparisons" % (P, ok))


if __name__ == "__main__":
    main()
