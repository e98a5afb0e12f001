"""
Survey bispectrum benchmark: ConvolvedFFTBispectrum of a LogNormalCatalog of 1e7 objects (L = 1000 Mpc/h) shifted
off the origin, with uniform randoms at 10x the density and a constant NZ, 32 shells up to the Nyquist wavenumber,
painted (CIC) to 256^3 in f8 and to 512^3 in f4, each with poles=[0] and poles=[0, 2, 4].

  python bench_convolved_bispectrum.py [--sizes 256f8,512f4] [--poles 0/0,2,4] [--warmup 0]

A 64^3 call with every multipole runs first, so that the timed calls do not load modules; --warmup adds full-size
calls.  Prints one JSON line: the card and its power limit (read in the same run); per workload and pole set the wall
time of one call, the CUDA-event stage times (paint, r2c, Y_lm, fills, c2r, triple sum, all-reduce), the transform
count and the peak device memory torch allocated during the call.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

NSHELL = 32
N_OBJECTS, BOX = 1e7, 1000.
SHIFT = np.array([1500., -700., 2300.])
SIZES = {"256f8": (256, "f8"), "512f4": (512, "f4")}


def _card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = out.stdout.strip() or "not read"
    except Exception:      # noqa: BLE001
        power = "not read"
    return name, power


def _fkp(n, L, seed=42):
    from nbodykit_b200.cosmology import NoWiggleEHPower
    from nbodykit_b200.lab import FKPCatalog, LogNormalCatalog, UniformCatalog
    nbar = n / L ** 3
    d = LogNormalCatalog(Plin=NoWiggleEHPower(), nbar=nbar, BoxSize=L, Nmesh=256, seed=seed)
    r = UniformCatalog(nbar=10 * nbar, BoxSize=L, seed=seed + 1)
    for c in (d, r):
        c['Position'] = c['Position'] + SHIFT
        c['NZ'] = nbar
    return FKPCatalog(d, r)


def _call(fkp, N, typestr, L, poles):
    from nbodykit_b200.lab import ConvolvedFFTBispectrum
    mesh = fkp.to_mesh(Nmesh=N, BoxSize=L, BoxCenter=SHIFT + L / 2, dtype=typestr, resampler="cic")
    return ConvolvedFFTBispectrum(mesh, poles=poles, dk=np.pi * N / L / NSHELL)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="256f8,512f4")
    ap.add_argument("--poles", default="0/0,2,4", help="pole sets separated by '/'")
    ap.add_argument("--warmup", type=int, default=0)
    args = ap.parse_args()
    pole_sets = [[int(v) for v in p.split(",")] for p in args.poles.split("/")]

    from nbodykit_b200 import _lib
    name, power = _card()
    res = dict(metric="convolved_bispectrum", gpus=1, card=name, power_limit=power, objects=N_OBJECTS,
               randoms=10 * N_OBJECTS, box=BOX, shells=NSHELL, resampler="cic", runs={})
    fkp = _fkp(N_OBJECTS, BOX)
    _call(_fkp(2e5, 500., seed=7), 64, "f8", 500., [0, 2, 4])           # loads the modules
    for size in args.sizes.split(","):
        N, typestr = SIZES[size]
        for poles in pole_sets:
            for _ in range(args.warmup):
                _call(fkp, N, typestr, BOX, poles)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            _lib.profiler.start()
            t0 = time.perf_counter()
            r = _call(fkp, N, typestr, BOX, poles)
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            stages = {k: round(sum(v), 3) for k, v in _lib.profiler.stop().items()}
            res["runs"]["%s/%s" % (size, ",".join(map(str, poles)))] = dict(
                Nmesh=N, dtype=typestr, poles=poles, seconds=round(wall, 4), stages_ms=stages,
                transforms=int(r.attrs["transforms"]), triangles=int(np.nansum(r.poles["triangles"])),
                peak_gib=round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 2),
                finite_B0=bool(np.isfinite(r.poles["B_0"][r.poles["triangles"] > 0]).all()))
            del r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
