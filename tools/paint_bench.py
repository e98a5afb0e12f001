"""Scratch: tiled paint timing on log-normal particles (generator order and randomly permuted), CUDA events."""
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nbodykit_b200.comm import SelfComm
from nbodykit_b200.cosmology import NoWiggleEHPower
from nbodykit_b200.pmesh.pm import ParticleMesh, RealField
from nbodykit_b200.source.catalog.lognormal import LogNormalCatalog


def timeit(fn, warm=2, rep=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(rep):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return min(ts), float(np.median(ts))


def main():
    npart = float(sys.argv[1]) if len(sys.argv) > 1 else 1e8
    Nmesh = int(sys.argv[2]) if len(sys.argv) > 2 else 512
    res = sys.argv[3] if len(sys.argv) > 3 else "cic"
    dtype = sys.argv[4] if len(sys.argv) > 4 else "f8"
    check = "--check" in sys.argv
    Box = 2.0 * Nmesh
    torch.cuda.set_device(0)
    cat = LogNormalCatalog(Plin=NoWiggleEHPower(), nbar=npart / Box ** 3, BoxSize=Box, Nmesh=Nmesh // 2, bias=2.0, seed=42,
                           comm=SelfComm())
    pos = cat['Position'].compute()
    del cat
    torch.cuda.empty_cache()
    n = pos.shape[0]
    pm = ParticleMesh(BoxSize=Box, Nmesh=Nmesh, dtype=dtype, comm=SelfComm())
    real = RealField(pm)
    alg = n * 12.0 + real.value.numel() * real.value.element_size()
    g = torch.Generator(device=pos.device); g.manual_seed(45)
    perm = torch.randperm(n, device=pos.device, generator=g)
    pp = pos[perm].contiguous()
    del perm
    ref = None
    cases = (("sorted", pos),) if "--only-sorted" in sys.argv else (("sorted", pos), ("permuted", pp))
    tag = " ".join("%s=%s" % (k[10:], v) for k, v in sorted(os.environ.items()) if k.startswith("NBK_PAINT_"))
    for label, p in cases:
        t = timeit(lambda: pm.paint(p, resampler=res, hold=False, out=real, method='tiled'))
        print("%s %d^3 %s n=%d %-8s [%s]: %.3f ms (median %.3f) -> %.3e part/s, %.0f GB/s algorithmic" % (
            res, Nmesh, dtype, n, label, tag, t[0], t[1], n / t[0] * 1e3, alg / t[0] / 1e6), flush=True)
        if ref is None:
            ref = real.value.clone()
            print("   sum = %.6f (n = %d)" % (real.csum(), n))
        else:
            print("   identical to the first mesh:", bool(torch.equal(ref, real.value)))
    if check:
        t = timeit(lambda: pm.paint(pos, resampler=res, hold=False, out=real, method='direct'), warm=1, rep=2)
        d = (real.value - ref).abs().max().item()
        print("direct: %.3f ms; max |tiled - direct| = %.3e (max cell %.3e)" % (t[0], d, ref.abs().max().item()))
        # hold=True (TMA reduce-add write-back) on top of the first mesh
        real.value.copy_(ref)
        pm.paint(pos, resampler=res, hold=True, out=real, method='tiled')
        d = (real.value - 2 * ref).abs().max().item()
        print("hold=True: max |2x - (x + x)| = %.3e" % d)


if __name__ == "__main__":
    main()
