"""
Fiber-collision benchmark: FiberCollisions on uniform skies at about 1000 and 4000 objects per square degree, the
reference test's field at 2e5 rows, and a clustered sky.

  python bench_fibercollisions.py [--sizes 1e6,1e7,1e8] [--densities 1000,4000] [--warmup 1]
  torchrun --nproc-per-node N bench_fibercollisions.py          (several GPUs, one process each)

Prints one JSON line: the card and its power limit (read in the same run), and per workload the wall time of the
constructor, the per-stage CUDA-event times (fof, route, sort, small groups, lists, greedy, nearest), the groups, the
largest group, the greedy steps, the collision-list entries, the collided rows and the peak device memory per row.
Workloads:
  field2e5   2e5 rows uniform in ra [0, 10), dec [-5, 0) (4000 per square degree; the reference test's field, 20 times
             denser), seed 42
  uniform    n rows uniform on a cap of the sky sized for the given density, for every --sizes and --densities
  clustered  --clustered-n rows: half uniform at 1000 per square degree, half in Gaussian clumps of 0.05 degrees
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

STAGES = ("fc_fof", "fc_route", "fc_sort", "fc_small", "fc_lists", "fc_greedy", "fc_nearest")


def _card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = out.stdout.strip() or "not read"
    except Exception:      # noqa: BLE001
        power = "not read"
    return name, power


def _cap(n, density, seed):
    """n rows uniform on the polar cap of area n / density square degrees (ra, dec in degrees, float64)"""
    area = n / float(density) * (np.pi / 180.) ** 2          # steradians
    zmin = 1.0 - area / (2 * np.pi)
    if zmin < -1:
        raise ValueError("%d rows at %g per square degree exceed the sky" % (n, density))
    g = torch.Generator(device="cuda").manual_seed(seed)
    ra = torch.rand(n, generator=g, device="cuda", dtype=torch.float64) * 360.
    z = zmin + (1 - zmin) * torch.rand(n, generator=g, device="cuda", dtype=torch.float64)
    dec = torch.rad2deg(torch.asin(z))
    return ra, dec


def _field2e5():
    np.random.seed(42)
    n = 200000
    return 10. * np.random.random(size=n), 5. * np.random.random(size=n) - 5.0


def _clustered(n, seed=45):
    ra, dec = _cap(n // 2, 1000., seed)
    rng = np.random.RandomState(seed)
    m = n - n // 2
    nclump = max(1, m // 2000)
    c = np.stack([rng.uniform(0, 360, nclump), np.rad2deg(np.arcsin(rng.uniform(np.sin(np.deg2rad(30.)), 1., nclump)))], 1)
    k = rng.randint(0, nclump, m)
    cra = c[k, 0] + rng.normal(scale=0.05, size=m) / np.cos(np.deg2rad(c[k, 1]))
    cdec = np.clip(c[k, 1] + rng.normal(scale=0.05, size=m), -90, 90)
    return (torch.cat([ra, torch.from_numpy(cra % 360.).cuda()]), torch.cat([dec, torch.from_numpy(cdec).cuda()]))


def _split(x, comm):
    n = int(x.shape[0])
    return x[comm.rank * n // comm.size:(comm.rank + 1) * n // comm.size]


def _run(ra, dec, comm, warmup):
    from nbodykit_b200._lib import profiler
    from nbodykit_b200.lab import FiberCollisions
    ra, dec = _split(ra, comm), _split(dec, comm)
    for _ in range(warmup):
        FiberCollisions(ra, dec, seed=1, comm=comm)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    profiler.start()
    t0 = time.perf_counter()
    r = FiberCollisions(ra, dec, seed=1, comm=comm)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    rec = profiler.stop()
    n = int(comm.allreduce(int(ra.shape[0])))
    s = r._stats
    out = dict(rows=n, wall_s=round(wall, 4),
               stages_ms={k[3:]: round(sum(rec.get(k, [0.0])), 3) for k in STAGES},
               groups=s['groups'], largest=int(comm.allreduce(s['largest'], op='max')) if comm.size > 1 else s['largest'],
               pairs=int(comm.allreduce(s['pairs'])), multiplets=int(comm.allreduce(s['multiplets'])),
               greedy_steps=int(comm.allreduce(s['steps'])), list_entries=int(comm.allreduce(s['list_entries'])),
               collided=int(comm.allreduce(s['collided'])),
               peak_bytes_per_row=round((torch.cuda.max_memory_allocated() - base) / max(1, int(ra.shape[0])), 1))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1e6,1e7,1e8")
    ap.add_argument("--densities", default="1000,4000")
    ap.add_argument("--clustered-n", type=float, default=1e7)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    from nbodykit_b200 import comm as C
    world = C.world() if int(os.environ.get("WORLD_SIZE", "1")) > 1 else C.SelfComm()
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    card, power = _card()
    res = dict(bench="fibercollisions", card=card, power_limit=power, gpus=world.size, workloads={})
    ra, dec = _field2e5()
    res["workloads"]["field2e5"] = _run(torch.from_numpy(ra).cuda(), torch.from_numpy(dec).cuda(), world, args.warmup)
    for d in [float(v) for v in args.densities.split(",")]:
        for n in [int(float(v)) for v in args.sizes.split(",")]:
            name = "uniform_%d_%g" % (d, n)
            try:
                ra, dec = _cap(n, d, 46)
            except ValueError as e:
                res["workloads"][name] = str(e)
                continue
            res["workloads"][name] = _run(ra, dec, world, args.warmup)
            del ra, dec
            torch.cuda.empty_cache()
    ra, dec = _clustered(int(args.clustered_n))
    res["workloads"]["clustered_%g" % args.clustered_n] = _run(ra, dec, world, args.warmup)
    if world.rank == 0:
        print(json.dumps(res))


if __name__ == "__main__":
    main()
