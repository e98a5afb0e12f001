"""
Friends-of-friends benchmark: FOF(linking_length=0.2, nmin=20) + find_features on a LogNormalCatalog.

  python bench_fof.py --n 1e8 [--oracle-n 1e6] [--warmup 1]
  torchrun --nproc-per-node N bench_fof.py --n 1e8          (several GPUs, one process each)

Prints one JSON line: the card and its power limit (read in the same run), per-stage CUDA-event times (keys, sort,
link, finalise, merge, labels, features), particles/s, halo count, peak memory, the CPU oracle's time next to the GPU
time at --oracle-n with exact partition parity, and a permuted-input partition check at the large size.
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
    Nmesh = int(min(1024, 2 ** round(np.log2(L / 2.0))))
    return LogNormalCatalog(Plin=NoWiggleEHPower(), nbar=nbar, BoxSize=L, Nmesh=Nmesh, seed=seed, comm=comm)


def _partition_equal(a, b):
    """same partition of the rows up to renaming of the labels (device tensors of labels, label 0 included)"""
    a, b = a.to(torch.int64), b.to(torch.int64)
    pairs = torch.unique(a * (int(b.max()) + 1) + b).numel()
    return pairs == torch.unique(a).numel() == torch.unique(b).numel()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=float, default=1e8)
    ap.add_argument("--oracle-n", type=float, default=1e6)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--no-permute", action="store_true")
    args = ap.parse_args()

    from nbodykit_b200 import _lib
    from nbodykit_b200.comm import SelfComm, world
    from nbodykit_b200.lab import ArrayCatalog, FOF
    comm = world()
    if torch.cuda.is_available():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    name, power = _card()
    res = dict(metric="fof", gpus=comm.size, card=name, power_limit=power)

    src = _catalog(args.n, comm)
    res["particles"] = int(src.csize)
    res["box"] = float(src.attrs["BoxSize"][0])
    for _ in range(args.warmup):
        FOF(src, linking_length=0.2, nmin=20).find_features()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base_mem = torch.cuda.memory_allocated()
    _lib.profiler.start()
    comm.barrier()
    t0 = time.perf_counter()
    fof = FOF(src, linking_length=0.2, nmin=20)
    feat = fof.find_features()
    torch.cuda.synchronize()
    comm.barrier()
    wall = time.perf_counter() - t0
    stages = {k: round(sum(v), 3) for k, v in _lib.profiler.stop().items() if k.startswith("fof")}
    res.update(seconds=round(wall, 4), particles_per_s=round(src.csize / wall, 1), stages_ms=stages,
               halos=int(max(fof.max_label)), merge_rounds=int(fof.merge_rounds),
               peak_mem_gb=round(torch.cuda.max_memory_allocated() / 1e9, 3),
               fof_mem_bytes_per_particle=round((torch.cuda.max_memory_allocated() - base_mem) / max(src.size, 1), 1),
               input_bytes_per_particle=24)
    del feat

    if comm.size == 1 and not args.no_permute:
        pos = src["Position"].compute()
        perm = torch.randperm(pos.shape[0], device=pos.device, generator=torch.Generator(device=pos.device).manual_seed(1))
        again = FOF(ArrayCatalog({"Position": pos[perm]}, comm=SelfComm(), BoxSize=src.attrs["BoxSize"]),
                    linking_length=0.2 * (np.prod(src.attrs["BoxSize"]) / src.csize) ** (1 / 3.), nmin=20, absolute=True)
        lab_a = torch.as_tensor(fof.labels, device=pos.device)[perm]
        lab_b = torch.as_tensor(again.labels, device=pos.device)
        res["permuted_partition_equal"] = bool(_partition_equal(lab_a, lab_b))
        res["permuted_sizes_equal"] = bool(torch.equal(torch.sort(torch.bincount(lab_a.long())[1:]).values,
                                                       torch.sort(torch.bincount(lab_b.long())[1:]).values))
        del pos, again

    if comm.size == 1 and args.oracle_n > 0:
        from oracle import fof_oracle as fo
        small = _catalog(args.oracle_n, SelfComm(), seed=7)
        p = small["Position"].compute().cpu().numpy()
        b = 0.2 * (np.prod(small.attrs["BoxSize"]) / small.csize) ** (1 / 3.)
        FOF(small, linking_length=0.2, nmin=20)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        g = FOF(small, linking_length=0.2, nmin=20)
        torch.cuda.synchronize()
        tg = time.perf_counter() - t0
        t0 = time.perf_counter()
        want = fo.fof_labels(p, b, 20, list(small.attrs["BoxSize"]))
        tc = time.perf_counter() - t0
        res["oracle"] = dict(particles=int(small.csize), gpu_s=round(tg, 4), cpu_oracle_s=round(tc, 3),
                             labels_identical=bool(np.array_equal(g.labels, want)))
    if comm.rank == 0:
        print(json.dumps(res))


if __name__ == "__main__":
    main()
