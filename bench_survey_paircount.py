"""
Survey pair-count benchmark: SurveyDataPairCount on a clustered survey shell (a LogNormalCatalog seen from the centre
of its box, 300 < r < 1000 Mpc/h, converted to RA / Dec / redshift with Planck15) in three workloads: '2d' with
Nmu = 100 and 'projected' with pimax = 80 (r / r_p edges: linspace(10, 150, 10)), and 'angular' with theta edges
logspace(-2, 0, 16) degrees.  In the same run SimulationBoxPairCount('2d', periodic=False) counts the same Cartesian
rows, and the survey / box ratio of the count kernel's time is reported.

  python bench_survey_paircount.py --n 1e6 [--oracle-n 3e4] [--warmup 1] [--modes 2d,projected,angular]

Prints one JSON line: the card and its power limit (read in the same run); per workload the wall time, the CUDA-event
stage times (sky transform, cells, route, count, reduce), pairs in range and candidate pairs tested, each per second;
the box '2d' count on the same rows and the count-kernel ratio; and an oracle comparison at --oracle-n with exact
npairs parity in every workload.
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

REDGES = np.linspace(10, 150, 10)
THETA = np.logspace(-2, 0, 16)
WORKLOADS = {"2d": (REDGES, dict(Nmu=100)), "projected": (REDGES, dict(pimax=80.)), "angular": (THETA, {})}
RMIN, RMAX, L = 300., 1000., 2000.


def _card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = out.stdout.strip() or "not read"
    except Exception:      # noqa: BLE001
        power = "not read"
    return name, power


def _shell(n, comm, seed=42):
    """an ArrayCatalog of RA, DEC, Redshift of about n objects in the shell RMIN < r < RMAX, and their Cartesian rows"""
    from nbodykit_b200 import transform as T
    from nbodykit_b200.cosmology import NoWiggleEHPower, Planck15
    from nbodykit_b200.lab import ArrayCatalog, LogNormalCatalog
    nbar = n / (4. / 3. * np.pi * (RMAX ** 3 - RMIN ** 3))
    Nmesh = int(min(512, 2 ** round(np.log2(L / 6.0))))
    src = LogNormalCatalog(Plin=NoWiggleEHPower(), nbar=nbar, BoxSize=L, Nmesh=Nmesh, seed=seed, comm=comm)
    pos = src["Position"].compute().double() - 0.5 * L
    r = torch.linalg.vector_norm(pos, dim=1)
    pos = pos[(r > RMIN) & (r < RMAX)]
    ra, dec, z = T.CartesianToSky(pos, Planck15)
    cat = ArrayCatalog({"RA": ra, "DEC": dec, "Redshift": z}, comm=comm)
    return cat, T.SkyToCartesian(ra, dec, z, Planck15)


def _timed(fn, warmup):
    from nbodykit_b200 import _lib
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    _lib.profiler.start()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    stages = {k.replace("paircount_", ""): round(sum(v), 3) for k, v in _lib.profiler.stop().items()
              if k.startswith("paircount")}
    return r, wall, stages


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=float, default=1e6)
    ap.add_argument("--oracle-n", type=float, default=3e4)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--modes", default="2d,projected,angular")
    args = ap.parse_args()

    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200.lab import ArrayCatalog, SimulationBoxPairCount, SurveyDataPairCount
    comm = SelfComm()
    torch.cuda.set_device(0)
    name, power = _card()
    res = dict(metric="survey_paircount", gpus=1, card=name, power_limit=power)

    cat, rows = _shell(args.n, comm)
    res["objects"] = int(cat.csize)
    res["shell_mpc_h"] = [RMIN, RMAX]
    res["workloads"] = {}
    for mode in args.modes.split(","):
        edges, kw = WORKLOADS[mode]
        r, wall, stages = _timed(lambda: SurveyDataPairCount(mode, cat, edges, cosmo=Planck15, **kw), args.warmup)
        pairs = int(r.pairs["npairs"].sum())
        cand = int(r.candidates)
        count_s = stages.get("count", float("nan")) / 1e3
        res["workloads"][mode] = dict(
            params=dict(kw, edges_max=float(edges[-1])), bins=int(np.prod(r.pairs.shape)), seconds=round(wall, 4),
            stages_ms=stages, pairs_in_range=pairs, candidates=cand, pairs_per_s=round(pairs / wall, 1),
            candidates_per_s_count_kernel=round(cand / count_s, 1), candidates_per_s_wall=round(cand / wall, 1))

    if "2d" in res["workloads"]:
        # the same rows as a non-periodic box: the count kernel without the per-pair line of sight
        box = ArrayCatalog({"Position": rows}, comm=comm, BoxSize=[2 * RMAX] * 3)
        b, wall, stages = _timed(lambda: SimulationBoxPairCount("2d", box, REDGES, periodic=False, Nmu=100),
                                 args.warmup)
        s = res["workloads"]["2d"]
        res["box_2d_same_rows"] = dict(seconds=round(wall, 4), stages_ms=stages,
                                       pairs_in_range=int(b.pairs["npairs"].sum()), candidates=int(b.candidates),
                                       npairs_total_equal=int(b.pairs["npairs"].sum()) == s["pairs_in_range"])
        res["survey_over_box_count_kernel_2d"] = round(s["stages_ms"]["count"] / stages["count"], 3)

    if args.oracle_n > 0:
        from oracle import survey_paircount_oracle as so
        small, srows = _shell(args.oracle_n, comm, seed=7)
        from nbodykit_b200 import transform as T
        unit = T.SkyToUnitSphere(small["RA"].compute(), small["DEC"].compute()).cpu().numpy()
        res["oracle"] = dict(objects=int(small.csize))
        for mode in args.modes.split(","):
            edges, kw = WORKLOADS[mode]
            g = SurveyDataPairCount(mode, small, edges, cosmo=Planck15, **kw)
            t0 = time.perf_counter()
            want = so.count(unit if mode == "angular" else srows.cpu().numpy(), mode, edges, **kw)
            res["oracle"][mode] = dict(cpu_oracle_s=round(time.perf_counter() - t0, 3),
                                       pairs=int(want["npairs"].sum()),
                                       npairs_identical=bool(np.array_equal(g.pairs["npairs"], want["npairs"])))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
