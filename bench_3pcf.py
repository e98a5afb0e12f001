"""
Three-point benchmark: SimulationBox3PCF on a LogNormalCatalog, the reference's benchmark workload (edges
linspace(0, 150, 9), l = 0 .. 10) at two sizes: boss_like (1e6 objects, L = 2500 Mpc/h) and desi_like (1e7, L = 5000).

  python bench_3pcf.py [--sizes boss_like,desi_like] [--warmup 1] [--oracle-n 2e4]
  torchrun --nproc-per-node N bench_3pcf.py                  (several GPUs, one process each)

Prints one JSON line: the card and its power limit (read in the same run); per size the wall time, the CUDA-event
stage times (cells, route, count, reduce), neighbour pairs in range and candidate pairs tested, each per second, and
an FP64 operation estimate over the H100 SXM data sheet's non-tensor FP64 rate (a data-sheet bound, not a measured
peak); the reference's golden C++ result through the GPU path; and an oracle comparison at --oracle-n objects (the
boss_like density, edges linspace(0, 40, 9), l = 0 .. 10) with the CPU oracle's time beside the GPU time.
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
EDGES = np.linspace(0, 150, 9)
POLES = list(range(11))
SIZES = {"boss_like": (1e6, 2500.), "desi_like": (1e7, 5000.)}


def fp64_ops(pairs, primaries, poles, nb):
    """FP64 operations of the count kernel: per pair in range the separation (3 differences, 3 squares, 2 additions,
    a square root, 3 divisions), the ladders (6 per power of ux + i uy, 1 per power of uz) and 4 per moment (two
    fma); per primary and bin 4 per table term of the moment -> a_lm conversion; per primary and (l, b1 <= b2) 4 per m
    of the outer product plus 2.  Square roots and divisions count as one operation each."""
    L = max(poles)
    nmom = (L + 1) * (L + 2) // 2
    per_pair = 12 + 7 * (L + 1) + 4 * nmom
    table_terms = sum((ell - m) // 2 + 1 for ell in range(L + 1) for m in range(ell + 1))
    nbp = nb * (nb + 1) // 2
    per_primary = 4 * table_terms * nb + sum(4 * (ell + 1) + 2 for ell in poles) * nbp
    return pairs * per_pair + primaries * per_primary


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
    Nmesh = int(min(512, 2 ** round(np.log2(L / 10.))))
    return LogNormalCatalog(Plin=NoWiggleEHPower(), nbar=n / L ** 3, BoxSize=L, Nmesh=Nmesh, seed=seed, comm=comm)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="boss_like,desi_like")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--oracle-n", type=float, default=2e4)
    args = ap.parse_args()

    from nbodykit_b200 import _lib
    from nbodykit_b200.comm import SelfComm, world
    from nbodykit_b200.lab import ArrayCatalog, SimulationBox3PCF
    comm = world()
    if torch.cuda.is_available():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    name, power = _card()
    res = dict(metric="threeptcf", gpus=comm.size, card=name, power_limit=power, edges=EDGES.tolist(), poles=POLES)
    res["sizes"] = {}
    for size in args.sizes.split(","):
        n, L = SIZES[size]
        src = _catalog(n, L, comm)
        for _ in range(args.warmup):
            SimulationBox3PCF(src, POLES, EDGES)
        torch.cuda.synchronize()
        _lib.profiler.start()
        comm.barrier()
        t0 = time.perf_counter()
        r = SimulationBox3PCF(src, POLES, EDGES)
        torch.cuda.synchronize()
        comm.barrier()
        wall = time.perf_counter() - t0
        stages = {k.replace("threeptcf_", ""): round(sum(v), 3) for k, v in _lib.profiler.stop().items()
                  if k.startswith("threeptcf")}
        pairs = int(r.npairs.sum())
        cand = int(r.candidates)
        count_s = stages.get("count", float("nan")) / 1e3
        ops = fp64_ops(pairs, int(src.csize), POLES, len(EDGES) - 1)
        res["sizes"][size] = dict(
            objects=int(src.csize), box=L, seconds=round(wall, 4), stages_ms=stages, pairs_in_range=pairs,
            candidates=cand, pairs_per_s_count_kernel=round(pairs / count_s, 1), pairs_per_s_wall=round(pairs / wall, 1),
            candidates_per_s_count_kernel=round(cand / count_s, 1), fp64_ops_estimate=float(ops),
            fp64_tflops_count_kernel=round(ops / count_s / 1e12, 3),
            datasheet_fp64_bound_fraction=round(ops / count_s / (DATASHEET_FP64 * comm.size), 4))
        del src, r

    if comm.size == 1:
        from oracle import threeptcf_oracle as to
        pos, w, truth = to.golden()
        cat = ArrayCatalog({"Position": torch.from_numpy(pos).cuda(), "w": torch.from_numpy(w).cuda()},
                           comm=SelfComm(), BoxSize=[400.] * 3)
        g = SimulationBox3PCF(cat, POLES, np.linspace(0, 200., 9), weight="w")
        rel = max(float(np.max(np.abs(g.poles["corr_%d" % ell] * (4 * np.pi) ** 2 / (2 * ell + 1) - truth[..., ell])
                               / np.abs(truth[..., ell]))) for ell in POLES)
        res["golden"] = dict(objects=len(pos), max_rel_vs_cpp=rel, passes_rtol_1e6=bool(rel <= 1e-6))

        if args.oracle_n > 0:
            n0, L0 = SIZES["boss_like"]
            Ls = float((args.oracle_n * L0 ** 3 / n0) ** (1 / 3.))
            small = _catalog(args.oracle_n, Ls, SelfComm(), seed=7)
            p = small["Position"].compute().cpu().numpy()
            edges = np.linspace(0, 40., 9)
            SimulationBox3PCF(small, POLES, edges)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            s = SimulationBox3PCF(small, POLES, edges)
            torch.cuda.synchronize()
            tg = time.perf_counter() - t0
            t0 = time.perf_counter()
            want = to.compute(p, edges, POLES, box=[Ls] * 3)
            tc = time.perf_counter() - t0
            z = np.stack([s.poles["corr_%d" % ell] for ell in POLES])
            res["oracle"] = dict(objects=int(small.csize), box=round(Ls, 3), edges=edges.tolist(), gpu_s=round(tg, 4),
                                 cpu_oracle_s=round(tc, 3), npairs_identical=bool(np.array_equal(s.npairs, want["npairs"])),
                                 max_err_over_bound=float(np.max(np.abs(z - want["zeta"]) / np.maximum(want["bound"], 1e-300))))
    if comm.rank == 0:
        print(json.dumps(res))


if __name__ == "__main__":
    main()
