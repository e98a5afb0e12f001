"""
Redshift histogram benchmark: RedshiftHistogram and its interpolation on N(0.5, 0.1) randoms.

  python bench_zhist.py [--n 1e9] [--oracle-n 1e7] [--reps 3] [--warmup 1]

Prints one JSON line: the card and its power limit (read in the same run), and per workload the per-stage CUDA-event
times (moments, bin, reduce, spline; mean of --reps runs after --warmup), the bytes the algorithm has to move, the rate
over the stage times and its share of the 3.35 TB/s data-sheet HBM3 bandwidth of the H100 SXM; then the NumPy / SciPy
oracle's time at --oracle-n rows with an output check.  Workloads (--n rows each):
  scott_f8, scott_f8_weighted   float64 redshifts (and float64 weights), Scott's rule: two passes over z
  scott_f4, scott_f4_weighted   the same in float32
  edges200                      200 non-uniform explicit edges: one pass (binary search, shared-memory histogram)
  edges_global                  20000 evenly spaced explicit edges, beyond the shared-memory histogram (global atomics)
  interpolate                   the spline of the scott_f8 histogram at every row: 8 B in and 8 B out per row
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

HBM_BYTES_PER_S = 3.35e12     # NVIDIA H100 SXM data sheet
STAGES = ("moments", "bin", "reduce", "spline")


def _card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = out.stdout.strip() or "not read"
    except Exception:      # noqa: BLE001
        power = "not read"
    return name, power


def _nonuniform_edges(nb):
    e = np.r_[0.0, np.cumsum(np.random.RandomState(nb).uniform(0.2, 1.8, nb))]
    return 0.0 + 1.0 * e / e[-1]


def _timed(fn, reps, warmup):
    from nbodykit_b200 import _lib
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    _lib.profiler.start()
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) / reps
    prof = _lib.profiler.stop()
    stages = {s: round(sum(prof.get("zh_" + s, [0.0])) / reps, 3) for s in STAGES}
    return out, stages, wall


def _report(stages, wall, nbytes, floor_ms):
    ms = sum(stages.values())
    rate = nbytes / (ms / 1e3) if ms > 0 else 0.0
    return dict(stages_ms=stages, stage_sum_ms=round(ms, 3), wall_ms=round(wall * 1e3, 3), bytes=int(nbytes),
                bytes_per_s=round(rate, 1), share_of_hbm_peak=round(rate / HBM_BYTES_PER_S, 3),
                data_sheet_floor_ms=round(floor_ms, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=float, default=1e9)
    ap.add_argument("--oracle-n", type=float, default=1e7)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()

    from nbodykit_b200 import _lib
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200.lab import ArrayCatalog, RedshiftHistogram
    torch.cuda.set_device(0)
    name, power = _card()
    n = int(args.n)
    res = dict(metric="zhist", rows=n, card=name, power_limit=power, hbm_data_sheet_bytes_per_s=HBM_BYTES_PER_S,
               smem_bins=int(_lib.lib().nbk_zh_smem_bins()), workloads={})
    g = torch.Generator(device="cuda").manual_seed(7)
    z8 = torch.randn(n, generator=g, device="cuda", dtype=torch.float64).mul_(0.1).add_(0.5)
    w8 = torch.rand(n, generator=g, device="cuda", dtype=torch.float64)

    def hist(z, w=None, bins=None):
        cols = {"z": z}
        if w is not None:
            cols["w"] = w
        return RedshiftHistogram(ArrayCatalog(cols, comm=SelfComm()), 0.15, Planck15, bins=bins, redshift="z",
                                 weight="w" if w is not None else None)

    def add(key, fn, nbytes, **extra):
        r, stages, wall = _timed(fn, args.reps, args.warmup)
        res["workloads"][key] = dict(_report(stages, wall, nbytes, nbytes / HBM_BYTES_PER_S * 1e3), **extra)
        return r

    r8 = add("scott_f8", lambda: hist(z8), 16 * n)
    res["workloads"]["scott_f8"]["bins"] = len(r8.bin_edges) - 1
    add("scott_f8_weighted", lambda: hist(z8, w8), 24 * n)
    z4, w4 = z8.float(), w8.float()
    add("scott_f4", lambda: hist(z4), 8 * n)
    add("scott_f4_weighted", lambda: hist(z4, w4), 12 * n)
    del z4, w4
    add("edges200", lambda: hist(z8, bins=_nonuniform_edges(200)), 8 * n, bins=200)
    add("edges_global", lambda: hist(z8, bins=np.linspace(0.0, 1.0, 20001)), 8 * n, bins=20000)
    del w8
    torch.cuda.empty_cache()
    add("interpolate", lambda: r8.interpolate(z8), 16 * n)
    del z8
    torch.cuda.empty_cache()

    if args.oracle_n > 0:
        from oracle import zhist_oracle as zo
        m = int(args.oracle_n)
        zs = zo.make_redshifts(11, m)
        t0 = time.perf_counter()
        o = zo.zhist(zs, 0.15, Planck15)
        oi = zo.interpolate(zs, o["bin_centers"], o["nbar"])
        tc = time.perf_counter() - t0
        zd = torch.from_numpy(zs).cuda()
        (r, ri), _, wall = _timed(lambda: (lambda h: (h, h.interpolate(zd)))(hist(zd)), 1, 1)
        same_edges = len(r.bin_edges) == len(o["bin_edges"]) and bool(np.allclose(r.bin_edges, o["bin_edges"], rtol=1e-13, atol=0))
        same_counts = bool(np.array_equal(r.nbar, zo.counts(zs, r.bin_edges) / r.dV))
        ri = ri.cpu().numpy()
        same_interp = bool(np.allclose(ri, zo.interpolate(zs, r.bin_centers, r.nbar), rtol=0, atol=1e-14 * r.nbar.max()))
        res["oracle"] = dict(rows=m, cpu_oracle_s=round(tc, 3), gpu_s=round(wall, 4), edges_within_1e13=same_edges,
                             counts_identical=same_counts, interpolation_within_1e14=same_interp,
                             oracle_interp_checked=bool(np.isfinite(oi).all()))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
