"""Tiled paint of the headline catalogue: tile-run statistics, per-kernel times and paint times per bucketing plan.

  python tools/paint_runs.py [--npart 1e9] [--order sorted|xsorted|random] [--stats] [--profile DIR]
                             [--time PLAN[,PLAN...]] [--reps 5]

--stats      mean length of the runs of consecutive particles with the same 16^3 tile (CIC leftmost cell), the share
             of particles in runs <= 2, and the run count once runs are also cut at 128-particle slices (what the run
             plan stores)
--profile    torch.profiler (CUDA activities) around 3 paints after a warm-up; kernel times per paint, to DIR
--time       CUDA-event paint times with NBK_PAINT_BUCKET set to each PLAN ("auto" = the probe's choice); every mesh is
             compared bit for bit with the first one
Orders: sorted = the generator's cell order; xsorted = sorted by x only (short runs, coherent planes); random.
"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:        # the numbers below are still valid, only unlabelled
        return "unknown (%s)" % e


def catalogue(npart, order):
    import bench
    cfg = dict(bench.CONFIGS["headline"])
    cfg["npart"] = npart
    pos = bench.generate(cfg, seed=42)
    if order == "random":
        g = torch.Generator(device=pos.device)
        g.manual_seed(45)
        pos = pos[torch.randperm(pos.shape[0], device=pos.device, generator=g)].contiguous()
    elif order == "xsorted":
        pos = pos[torch.sort(pos[:, 0], stable=True)[1]].contiguous()
    torch.cuda.empty_cache()
    return pos, cfg


def run_stats(pm, pos):
    n = pos.shape[0]
    c = pm.cell_index(pos, "cic")
    nt = [int(v) // 16 for v in pm.Nmesh]
    t = ((c[:, 0] // 16) * nt[1] + c[:, 1] // 16) * nt[2] + c[:, 2] // 16
    del c
    head = torch.ones(n, dtype=torch.bool, device=pos.device)
    head[1:] = t[1:] != t[:-1]
    hidx = torch.nonzero(head).squeeze(1)
    lens = torch.diff(torch.cat([hidx, torch.tensor([n], device=pos.device)]))
    nruns = int(hidx.numel())
    short = int(lens[lens <= 2].sum())
    head[::128] = True                           # runs are also cut at the 128-particle slices of a warp
    ncap = int(head.sum())
    pairs = float((t[1:] == t[:-1]).float().mean())
    print("runs: n = %d, runs = %d, mean run = %.3f, particles in runs <= 2: %.4f, runs cut at 128: %d (mean %.3f), "
          "equal-tile neighbour pairs: %.4f" % (n, nruns, n / nruns, short / n, ncap, n / ncap, pairs), flush=True)


def paint(pm, pos, real):
    pm.paint(pos, resampler="cic", hold=False, out=real, method="tiled")


def profile(pm, pos, real, outdir):
    from torch.profiler import ProfilerActivity, profile as tprof
    for _ in range(2):
        paint(pm, pos, real)
    torch.cuda.synchronize()
    reps = 3
    with tprof(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(reps):
            paint(pm, pos, real)
        torch.cuda.synchronize()
    tot = {}
    for e in p.key_averages():
        if e.device_type.name == "CUDA" and e.self_device_time_total > 0:
            tot[e.key] = (e.self_device_time_total / 1e3 / reps, e.count // reps)
    s = sum(v[0] for v in tot.values())
    for k, (ms, c) in sorted(tot.items(), key=lambda kv: -kv[1][0]):
        print("  %8.3f ms  x%-3d %s" % (ms, c, k[:150]), flush=True)
    print("  %8.3f ms  total per paint" % s, flush=True)
    os.makedirs(outdir, exist_ok=True)
    with open(os.path.join(outdir, "paint_kernels.txt"), "w") as f:
        f.write(p.key_averages().table(sort_by="self_device_time_total", row_limit=40))


def time_plans(pm, pos, real, plans, reps):
    ref = None
    for plan in plans:
        if plan == "auto":
            os.environ.pop("NBK_PAINT_BUCKET", None)
        else:
            os.environ["NBK_PAINT_BUCKET"] = plan
        for _ in range(2):
            paint(pm, pos, real)
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            paint(pm, pos, real)
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        same = ""
        if ref is None:
            ref = real.value.clone()
        else:
            same = ", mesh identical to %s's: %s" % (plans[0], bool(torch.equal(ref, real.value)))
        print("  plan %-9s paint %.3f ms (min %.3f, max %.3f over %d)%s" % (plan, float(np.median(ts)), min(ts), max(ts),
                                                                          reps, same), flush=True)
    os.environ.pop("NBK_PAINT_BUCKET", None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--npart", type=float, default=1e9)
    ap.add_argument("--order", default="sorted", choices=["sorted", "xsorted", "random"])
    ap.add_argument("--stats", action="store_true")
    ap.add_argument("--profile", metavar="DIR", default=None)
    ap.add_argument("--time", default=None)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.pmesh.pm import ParticleMesh, RealField
    print("GPU: %s" % gpu_info(), flush=True)
    pos, cfg = catalogue(args.npart, args.order)
    print("catalogue: %d particles, order %s" % (pos.shape[0], args.order), flush=True)
    pm = ParticleMesh(BoxSize=cfg["box"], Nmesh=cfg["nmesh"], dtype=cfg["dtype"], comm=SelfComm())
    if args.stats:
        run_stats(pm, pos)
    real = RealField(pm)
    if args.profile:
        profile(pm, pos, real, args.profile)
    if args.time:
        time_plans(pm, pos, real, args.time.split(","), args.reps)


if __name__ == "__main__":
    main()
