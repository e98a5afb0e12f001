"""
Bispectrum benchmark: FFTBispectrum of a LogNormalCatalog of 1e7 objects (L = 1000 Mpc/h) with 32 shells up to the
Nyquist wavenumber, painted to 256^3 in f8 and to 512^3 in f4.

  python bench_bispectrum.py [--sizes 256f8,512f4] [--warmup 1]
  torchrun --nproc-per-node N bench_bispectrum.py               (several GPUs, one process each)

Prints one JSON line: the card and its power limit (read in the same run); per workload the wall time, the CUDA-event
stage times (fill, c2r, triple sum, all-reduce), the c2r count and triangles evaluated; the triple-sum FLOPs over the
H100 SXM data sheet's non-tensor FP64 rate (the products are formed in float64 for both precisions) and the fill bytes
over its HBM3 bandwidth -- data-sheet bounds, not measured peaks; and the agreement with the float64 oracle at 64^3.
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

# NVIDIA H100 SXM data sheet (up to 700 W): 34 TFLOP/s FP64 without tensor cores, 3.35 TB/s HBM3
DATASHEET_FP64 = 34e12
DATASHEET_HBM = 3.35e12
NSHELL = 32
N_OBJECTS, BOX = 1e7, 1000.
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


def _catalog(n, L, comm, seed=42):
    from nbodykit_b200.cosmology import NoWiggleEHPower
    from nbodykit_b200.lab import LogNormalCatalog
    return LogNormalCatalog(Plin=NoWiggleEHPower(), nbar=n / L ** 3, BoxSize=L, Nmesh=256, seed=seed, comm=comm)


def fill_bytes(N, P, typestr, transforms_per_pass, fill_chunk):
    """HBM bytes of the fill kernels of one call on one rank: the I pass reads the complex slab once per fill call and
    writes one complex slab per shell; the J pass writes one complex f8 slab per shell and reads nothing"""
    cslab = N * N * (N // 2 + 1) // P
    isz = 8 if typestr == "f4" else 16
    calls = -(-transforms_per_pass // fill_chunk)
    return cslab * (isz * (calls + transforms_per_pass) + 16 * transforms_per_pass)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="256f8,512f4")
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()

    from nbodykit_b200 import _lib
    from nbodykit_b200.algorithms import bispectrum as bs
    from nbodykit_b200.comm import SelfComm, world
    from nbodykit_b200.lab import FFTBispectrum
    comm = world()
    if torch.cuda.is_available():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    name, power = _card()
    res = dict(metric="bispectrum", gpus=comm.size, card=name, power_limit=power, objects=N_OBJECTS, box=BOX,
               shells=NSHELL, bounds=dict(triple_sum="FP64 non-tensor, 34 TFLOP/s (data sheet)",
                                          fill="HBM3, 3.35 TB/s (data sheet)"))
    res["sizes"] = {}
    src = _catalog(N_OBJECTS, BOX, comm)
    for size in args.sizes.split(","):
        N, typestr = SIZES[size]
        mesh = src.to_mesh(Nmesh=N, BoxSize=BOX, resampler="cic", compensated=True, dtype=typestr)
        dk = np.pi * N / BOX / NSHELL
        for _ in range(args.warmup):
            FFTBispectrum(mesh, dk=dk)
        torch.cuda.synchronize()
        _lib.profiler.start()
        comm.barrier()
        t0 = time.perf_counter()
        r = FFTBispectrum(mesh, dk=dk)
        torch.cuda.synchronize()
        comm.barrier()
        wall = time.perf_counter() - t0
        stages = {k.replace("bispec_", ""): round(sum(v), 3) for k, v in _lib.profiler.stop().items()
                  if k.startswith("bispec_")}
        kedges = r.bispec.edges["k1"]
        ntri = len(bs.shell_triples(kedges))
        flops = 2 * 2 * float(N) ** 3 / comm.size * ntri * 2          # 2 FMAs per cell and triple, both passes
        tsum_s = stages.get("triple_sum", float("nan")) / 1e3
        fill_s = stages.get("fill", float("nan")) / 1e3
        fbytes = fill_bytes(N, comm.size, typestr, r.attrs["transforms"] // 2, bs._FILL_CHUNK)
        res["sizes"][size] = dict(
            Nmesh=N, dtype=typestr, seconds=round(wall, 4), stages_ms=stages, c2r=int(r.attrs["transforms"]),
            triples_evaluated=ntri, triangles=int(r.bispec["triangles"].sum()),
            triple_sum_flops=flops, triple_sum_tflops=round(flops / tsum_s / 1e12, 3),
            triple_sum_fp64_bound_fraction=round(flops / tsum_s / DATASHEET_FP64, 4),
            fill_bytes=fbytes, fill_tb_per_s=round(fbytes / fill_s / 1e12, 3),
            fill_hbm_bound_fraction=round(fbytes / fill_s / DATASHEET_HBM, 4))
        del mesh, r
    del src

    if comm.size == 1:
        from oracle import bispectrum_oracle as bo
        small = _catalog(2e5, 500., SelfComm(), seed=7)
        mesh = small.to_mesh(Nmesh=64, BoxSize=500., resampler="cic", compensated=True, dtype="f8")
        dk = 2 * 2 * np.pi / 500.
        r = FFTBispectrum(mesh, dk=dk)
        half = mesh.compute(mode="complex").numpy()
        kedges = r.bispec.edges["k1"]
        want = bo.fft_form(half, [64] * 3, [500.] * 3, kedges)
        i, j, l = want["triples"].T
        ok = want["triangles"] > 0
        err = np.abs(r.bispec["B"][i, j, l] - want["B"])[ok] / want["bound"][ok]
        same = bool(np.array_equal(r.bispec["triangles"][i, j, l], want["triangles"]))
        res["oracle"] = dict(Nmesh=64, shells=len(kedges) - 1, triples=len(want["triples"]), triangles_identical=same,
                             max_err_over_bound=float(err.max()),
                             agreement="ok" if same and err.max() <= 1e-10 else "FAILED")
    if comm.rank == 0:
        print(json.dumps(res))


if __name__ == "__main__":
    main()
