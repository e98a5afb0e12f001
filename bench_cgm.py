"""
Cylindrical-groups benchmark: CylindricalGroups on the reference test's catalogue and on a LogNormalCatalog.

  python bench_cgm.py [--n 1e7] [--oracle-n 2e4] [--warmup 1]
  torchrun --nproc-per-node N bench_cgm.py --n 1e7          (several GPUs, one process each)

Prints one JSON line: the card and its power limit (read in the same run), and per workload the per-stage CUDA-event
times (priority, route, cells, lists, rounds, assign, labels), rounds, centrals, satellites, higher-priority neighbours
per row, candidate pairs tested per second of the list passes, peak memory per row, and the CPU oracle's time at
--oracle-n rows with identical outputs.  Workloads:
  reference  UniformCatalog(3e-4, 256, seed=42), rperp = rpar = 10, ranked by a uniform log-mass, periodic, los z
  thin       LogNormalCatalog of --n objects ranked by a random log-mass, rperp = 1, rpar = 10, periodic, los z
  thick      the same at rperp = rpar = 10
  rowrank    the same at rperp = rpar = 10 with rankby=None: the catalogue is stored in cell order, so the priority
             follows position, which makes long dependency chains
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

STAGES = ("priority", "route", "cells", "lists", "rounds", "assign", "labels")


def _card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = out.stdout.strip() or "not read"
    except Exception:      # noqa: BLE001
        power = "not read"
    return name, power


def _lognormal(n, comm, seed=42):
    from nbodykit_b200.cosmology import NoWiggleEHPower
    from nbodykit_b200.lab import LogNormalCatalog
    nbar = 3e-4
    L = float((n / nbar) ** (1 / 3.))
    Nmesh = int(min(1024, 2 ** round(np.log2(L / 8.0))))
    src = LogNormalCatalog(Plin=NoWiggleEHPower(), nbar=nbar, BoxSize=L, Nmesh=Nmesh, seed=seed, comm=comm)
    rng = np.random.RandomState(seed * 1000 + comm.rank)
    src['logmass'] = torch.from_numpy(rng.uniform(12, 15, size=src.size)).cuda()
    return src


def _reference(comm):
    from nbodykit_b200.lab import UniformCatalog
    src = UniformCatalog(3e-4, BoxSize=256, seed=42, comm=comm)
    src['logmass'] = src.rng.uniform(12, 15)
    return src


def _run(src, rankby, rperp, rpar, warmup):
    from nbodykit_b200 import _lib
    from nbodykit_b200.lab import CylindricalGroups
    comm = src.comm
    kw = dict(rankby=rankby, rperp=rperp, rpar=rpar, flat_sky_los=[0, 0, 1], periodic=True)
    for _ in range(warmup):
        CylindricalGroups(src, **kw)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base_mem = torch.cuda.memory_allocated()
    _lib.profiler.start()
    comm.barrier()
    t0 = time.perf_counter()
    r = CylindricalGroups(src, **kw)
    torch.cuda.synchronize()
    comm.barrier()
    wall = time.perf_counter() - t0
    prof = _lib.profiler.stop()
    stages = {s: round(sum(prof.get("cgm_" + s, [0.0])), 3) for s in STAGES}
    types = np.asarray(r.groups['cgm_type'].compute())
    cen = int(comm.allreduce(int((types == 0).sum())))
    sat = int(comm.allreduce(int((types == 1).sum())))
    nb = int(comm.allreduce(int(r._stats['neighbours'])))
    cand = int(comm.allreduce(int(r._stats['candidates'])))
    lists_s = max(stages["lists"], 1e-6) / 1e3
    return r, dict(rows=int(src.csize), rperp=rperp, rpar=rpar, rankby=rankby, seconds=round(wall, 4), stages_ms=stages,
                   rounds=int(r.rounds), centrals=cen, satellites=sat, neighbours_per_row=round(nb / max(src.csize, 1), 3),
                   candidates_per_s=round(cand / lists_s, 1),
                   peak_mem_bytes_per_row=round((torch.cuda.max_memory_allocated() - base_mem) / max(src.size, 1), 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=float, default=1e7)
    ap.add_argument("--oracle-n", type=float, default=2e4)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()

    from nbodykit_b200.comm import SelfComm, world
    comm = world()
    if torch.cuda.is_available():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    name, power = _card()
    res = dict(metric="cgm", gpus=comm.size, card=name, power_limit=power, workloads={})

    _, res["workloads"]["reference"] = _run(_reference(comm), "logmass", 10., 10., args.warmup)
    src = _lognormal(args.n, comm)
    res["box"] = float(src.attrs["BoxSize"][0])
    _, res["workloads"]["thin"] = _run(src, "logmass", 1., 10., args.warmup)
    _, res["workloads"]["thick"] = _run(src, "logmass", 10., 10., args.warmup)
    _, res["workloads"]["rowrank"] = _run(src, None, 10., 10., args.warmup)
    del src

    if comm.size == 1 and args.oracle_n > 0:
        from oracle import cgm_oracle as co
        small = _lognormal(args.oracle_n, SelfComm(), seed=7)
        L = float(small.attrs["BoxSize"][0])
        r, info = _run(small, "logmass", 10., 10., 1)
        tg = info["seconds"]
        pos = small["Position"].compute().cpu().numpy()
        lm = small["logmass"].compute().cpu().numpy()
        t0 = time.perf_counter()
        t, h, s, _ = co.cgm(pos, [lm], 10., 10., los=[0, 0, 1], periodic=True, BoxSize=L)
        tc = time.perf_counter() - t0
        same = all(np.array_equal(np.asarray(r.groups[c].compute()), w)
                   for c, w in (("cgm_type", t), ("cgm_haloid", h), ("num_cgm_sats", s)))
        res["oracle"] = dict(rows=int(small.csize), gpu_s=tg, cpu_oracle_s=round(tc, 3), outputs_identical=bool(same))
    if comm.rank == 0:
        print(json.dumps(res))


if __name__ == "__main__":
    main()
