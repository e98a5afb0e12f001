"""
The fused x pass and binning (k_fft_x_bin) on the smallest ring it runs with: R + 1 slots of 64 x 8 modes, where the
k edges, their accumulators and the staged powers leave room for no more (256^3 at dk = 0.15 kf: 570 edges; 512^3 at
dk = 0.5 kf: 342 edges).  The combine frees a tile's R slots before its DFT, so the next tile's boxes then take every
slot of the ring.  Compared with the general path as in test_gpu_fused_xbin.
"""
import pytest

from test_gpu_fused_xbin import _run

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("nmesh,dk", [((256, 256, 256), 0.15), ((512, 512, 512), 0.5)])
def test_fused_smallest_ring(cuda, nmesh, dk):
    _run(nmesh, "f8", "cic", dk)
