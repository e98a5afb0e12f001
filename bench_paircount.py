"""
Pair-count benchmark: SimulationBoxPairCount on a LogNormalCatalog in three workloads, '1d' to 150 Mpc/h, '2d' with
Nmu = 100 and 'projected' with pimax = 80 (r / r_p edges: the reference's linspace(10, 150, 10)).

  python bench_paircount.py --n 1e7 [--oracle-n 3e4] [--warmup 1] [--modes 1d,2d,projected]
  torchrun --nproc-per-node N bench_paircount.py --n 1e7          (several GPUs, one process each)

Prints one JSON line: the card and its power limit (read in the same run); per workload the wall time, the CUDA-event
stage times (cells, route, count, reduce), pairs in range and candidate pairs tested, each per second, and the
candidate rate over the H100 SXM data sheet's non-tensor FP64 rate (a data-sheet bound, not a measured peak); and an
oracle comparison at --oracle-n with exact npairs parity and the CPU oracle's time beside the GPU time.
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

# NVIDIA H100 SXM data sheet: 34 TFLOP/s FP64 without tensor cores (at up to 700 W)
DATASHEET_FP64 = 34e12
# FP64 operations per candidate pair in the count kernel: 3 differences, 3 squares, 2 additions, and in a periodic box
# 3 more differences (L - |d|)
FLOPS_PER_CANDIDATE = {True: 11, False: 8}
REDGES = np.linspace(10, 150, 10)
WORKLOADS = {"1d": {}, "2d": dict(Nmu=100), "projected": dict(pimax=80.)}


def _card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = out.stdout.strip() or "not read"
    except Exception:      # noqa: BLE001
        power = "not read"
    return name, power


def _catalog(n, comm, seed=42):
    from nbodykit_b200.cosmology import NoWiggleEHPower
    from nbodykit_b200.lab import LogNormalCatalog
    nbar = 3e-3
    L = float((n / nbar) ** (1 / 3.))
    Nmesh = int(min(512, 2 ** round(np.log2(L / 4.0))))
    return LogNormalCatalog(Plin=NoWiggleEHPower(), nbar=nbar, BoxSize=L, Nmesh=Nmesh, seed=seed, comm=comm)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=float, default=1e7)
    ap.add_argument("--oracle-n", type=float, default=3e4)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--modes", default="1d,2d,projected")
    args = ap.parse_args()

    from nbodykit_b200 import _lib
    from nbodykit_b200.comm import SelfComm, world
    from nbodykit_b200.lab import SimulationBoxPairCount
    comm = world()
    if torch.cuda.is_available():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    name, power = _card()
    res = dict(metric="paircount", gpus=comm.size, card=name, power_limit=power)

    src = _catalog(args.n, comm)
    res["objects"] = int(src.csize)
    res["box"] = float(src.attrs["BoxSize"][0])
    res["workloads"] = {}
    for mode in args.modes.split(","):
        kw = WORKLOADS[mode]
        for _ in range(args.warmup):
            SimulationBoxPairCount(mode, src, REDGES, **kw)
        torch.cuda.synchronize()
        _lib.profiler.start()
        comm.barrier()
        t0 = time.perf_counter()
        r = SimulationBoxPairCount(mode, src, REDGES, **kw)
        torch.cuda.synchronize()
        comm.barrier()
        wall = time.perf_counter() - t0
        stages = {k.replace("paircount_", ""): round(sum(v), 3) for k, v in _lib.profiler.stop().items()
                  if k.startswith("paircount")}
        pairs = int(r.pairs["npairs"].sum())
        cand = int(r.candidates)
        count_s = stages.get("count", float("nan")) / 1e3
        rate = cand / count_s
        res["workloads"][mode] = dict(
            params=dict(kw, rmax=float(REDGES[-1])), bins=int(np.prod(r.pairs.shape)), seconds=round(wall, 4),
            stages_ms=stages, pairs_in_range=pairs, candidates=cand, pairs_per_s=round(pairs / wall, 1),
            candidates_per_s_count_kernel=round(rate, 1), candidates_per_s_wall=round(cand / wall, 1),
            datasheet_fp64_bound_fraction=round(rate * FLOPS_PER_CANDIDATE[True] / (DATASHEET_FP64 * comm.size), 4))

    if comm.size == 1 and args.oracle_n > 0:
        from oracle import paircount_oracle as po
        small = _catalog(args.oracle_n, SelfComm(), seed=7)
        p = small["Position"].compute().cpu().numpy()
        L = float(small.attrs["BoxSize"][0])
        edges = np.linspace(2., min(40., 0.45 * L), 10)
        SimulationBoxPairCount("2d", small, edges, Nmu=10)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        g = SimulationBoxPairCount("2d", small, edges, Nmu=10)
        torch.cuda.synchronize()
        tg = time.perf_counter() - t0
        t0 = time.perf_counter()
        want = po.count(p, "2d", edges, [L] * 3, Nmu=10)
        tc = time.perf_counter() - t0
        res["oracle"] = dict(objects=int(small.csize), mode="2d", gpu_s=round(tg, 4), cpu_oracle_s=round(tc, 3),
                             npairs_identical=bool(np.array_equal(g.pairs["npairs"], want["npairs"])),
                             wnpairs_max_rel=float(np.max(np.abs(g.pairs["wnpairs"] - want["wnpairs"])
                                                          / np.maximum(want["wnpairs"], 1e-300))))
    if comm.rank == 0:
        print(json.dumps(res))


if __name__ == "__main__":
    main()
