"""
Nearest-neighbour density benchmark: KDDensity on the reference test's catalogue, a uniform catalogue, a
LogNormalCatalog and a catalogue of dense clumps.

  python bench_kddensity.py [--n 1e7] [--uniform-n 1e8] [--oracle-n 1e5] [--rows-per-cell 1,2,4,8] [--warmup 1]
  torchrun --nproc-per-node N bench_kddensity.py --n 1e7          (several GPUs, one process each)

Prints one JSON line: the card and its power limit (read in the same run), and per workload the per-stage CUDA-event
times (unit, route, cells, self, phase2, back, density), candidate rows tested per row and per second of the walk,
the rows that needed phase 2 (several GPUs), peak memory per row, and the same workload at every --rows-per-cell; then the
CPU oracle's time at --oracle-n rows with an identical-output check.  Workloads:
  reference  LogNormalCatalog(nbar 3e-4, BoxSize 64, Nmesh 16, seed 42) of the reference's test
  uniform    UniformCatalog of about --uniform-n rows
  lognormal  LogNormalCatalog of --n rows (nbar 3e-4)
  clumps     --n / 10 uniform rows plus 20 Gaussian clumps of --n / 1000 rows each (sigma 0.02 mean separations), so that
             one cell holds thousands of rows
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

STAGES = ("unit", "route", "cells", "self", "phase2", "back", "density")


def _card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = out.stdout.strip() or "not read"
    except Exception:      # noqa: BLE001
        power = "not read"
    return name, power


def _lognormal(n, comm, seed=42, L=None, Nmesh=None):
    from nbodykit_b200.cosmology import NoWiggleEHPower
    from nbodykit_b200.lab import LogNormalCatalog
    nbar = 3e-4
    L = float((n / nbar) ** (1 / 3.)) if L is None else L
    Nmesh = int(min(1024, 2 ** round(np.log2(L / 8.0)))) if Nmesh is None else Nmesh
    return LogNormalCatalog(Plin=NoWiggleEHPower(), nbar=nbar, BoxSize=L, Nmesh=Nmesh, seed=seed, comm=comm)


def _uniform(n, comm):
    from nbodykit_b200.lab import UniformCatalog
    L = 1000.
    return UniformCatalog(n / L ** 3, BoxSize=L, seed=43, comm=comm)


def _clumps(n, comm, seed=44):
    from nbodykit_b200.lab import ArrayCatalog
    L = 1000.
    P, rank = comm.size, comm.rank
    rng = np.random.RandomState(seed)
    centres = rng.uniform(size=(20, 3)) * L
    sigma = 0.02 * L / n ** (1 / 3.)
    g = torch.Generator(device="cuda").manual_seed(seed * 100 + rank)
    nb, nc = int(n // 10) // P, int(n // 1000) // P
    parts = [torch.rand((nb, 3), generator=g, device="cuda", dtype=torch.float64) * L]
    for c in centres:
        parts.append(torch.from_numpy(c).cuda() + torch.randn((nc, 3), generator=g, device="cuda", dtype=torch.float64) * sigma)
    pos = torch.remainder(torch.cat(parts), L)
    return ArrayCatalog({"Position": pos}, comm=comm, BoxSize=L)


def _run(src, warmup, margin=1.0):
    from nbodykit_b200 import _lib
    from nbodykit_b200.lab import KDDensity
    comm = src.comm
    for _ in range(warmup):
        KDDensity(src, margin=margin)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base_mem = torch.cuda.memory_allocated()
    _lib.profiler.start()
    comm.barrier()
    t0 = time.perf_counter()
    r = KDDensity(src, margin=margin)
    torch.cuda.synchronize()
    comm.barrier()
    wall = time.perf_counter() - t0
    prof = _lib.profiler.stop()
    stages = {s: round(sum(prof.get("kd_" + s, [0.0])), 3) for s in STAGES}
    cand = int(comm.allreduce(int(r._stats['candidates'])))
    walk_s = max(stages["self"] + stages["phase2"], 1e-6) / 1e3
    N = max(int(src.csize), 1)
    return r, dict(rows=int(src.csize), ncell=int(r._stats['ncell']), seconds=round(wall, 4), stages_ms=stages,
                   candidates_per_row=round(cand / N, 2), candidates_per_s=round(cand / walk_s, 1),
                   phase2_rows=int(comm.allreduce(int(r._stats['phase2_rows']))),
                   phase2_queries=int(comm.allreduce(int(r._stats['phase2_queries']))),
                   peak_mem_bytes_per_row=round((torch.cuda.max_memory_allocated() - base_mem) / max(src.size, 1), 1))


def _sweep(src, rows_per_cell, warmup):
    """the workload at each cell size (rows per cell at the mean density)"""
    from nbodykit_b200.algorithms import kdtree
    keep = kdtree._ROWS_PER_CELL
    out = {}
    try:
        for m in rows_per_cell:
            kdtree._ROWS_PER_CELL = m
            _, info = _run(src, warmup)
            out[str(m)] = dict(ncell=info["ncell"], seconds=info["seconds"], walk_ms=info["stages_ms"]["self"],
                               cells_ms=info["stages_ms"]["cells"], candidates_per_row=info["candidates_per_row"])
    finally:
        kdtree._ROWS_PER_CELL = keep
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=float, default=1e7)
    ap.add_argument("--uniform-n", type=float, default=1e8)
    ap.add_argument("--oracle-n", type=float, default=1e5)
    ap.add_argument("--rows-per-cell", default="1,2,4,8")
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    rpc = [float(v) for v in args.rows_per_cell.split(",") if v]

    from nbodykit_b200.comm import SelfComm, world
    comm = world()
    if torch.cuda.is_available():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    name, power = _card()
    res = dict(metric="kddensity", gpus=comm.size, card=name, power_limit=power, workloads={})

    _, res["workloads"]["reference"] = _run(_lognormal(0, comm, L=64., Nmesh=16), args.warmup)
    for wl, make in (("uniform", lambda: _uniform(args.uniform_n, comm)), ("lognormal", lambda: _lognormal(args.n, comm)),
                     ("clumps", lambda: _clumps(args.n, comm))):
        src = make()
        _, res["workloads"][wl] = _run(src, args.warmup)
        if wl != "clumps" and rpc:
            res["workloads"][wl]["rows_per_cell"] = _sweep(src, rpc, args.warmup)
        if comm.size > 1:
            res["workloads"][wl]["phase2_rows_margin0"] = _run(src, 0, margin=0.0)[1]["phase2_rows"]
        del src
        torch.cuda.empty_cache()

    if comm.size == 1 and args.oracle_n > 0:
        from oracle import kddensity_oracle as ko
        small = _lognormal(args.oracle_n, SelfComm(), seed=7)
        L = float(small.attrs["BoxSize"][0])
        r, info = _run(small, 1)
        pos = small["Position"].compute().cpu().numpy()
        t0 = time.perf_counter()
        d, dens = ko.density(pos, L)
        tc = time.perf_counter() - t0
        same = bool(np.array_equal(r._distance, d) and np.allclose(r.density, dens, rtol=1e-15, atol=0))
        res["oracle"] = dict(rows=int(small.csize), gpu_s=info["seconds"], cpu_oracle_s=round(tc, 3),
                             distances_identical=bool(np.array_equal(r._distance, d)), outputs_identical=same)
    if comm.rank == 0:
        print(json.dumps(res))


if __name__ == "__main__":
    main()
