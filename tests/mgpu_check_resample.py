"""
Multi-GPU parity check of Fourier-space resampling, run under torchrun (one rank per GPU):
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29523 tests/mgpu_check_resample.py
ArrayMesh(...).compute(mode='real' / 'complex', Nmesh=M) and preview(Nmesh=M) on P GPUs, gathered, must equal the
single-GPU result computed on rank 0, to 1e-12 of the largest value (f8), at 48 -> 36, 32 -> 48 and 30 -> 42 (odd
halves of the slabs at P = 2: 15 and 21 rows).
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from nbodykit_b200 import CurrentMPIComm
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ArrayMesh
    comm = CurrentMPIComm.get()
    assert comm.size == world
    ok = True
    for Ns, M in [(48, 36), (32, 48), (30, 42)]:
        a = np.random.RandomState(Ns).standard_normal((Ns, Ns, Ns))
        mesh = ArrayMesh(a, BoxSize=64., comm=comm)
        got = {}
        for mode in ("real", "complex"):
            f = mesh.compute(mode=mode, Nmesh=M).numpy()
            parts = comm.allgather(f if mode == "real" else f.transpose(1, 0, 2))
            got[mode] = np.concatenate(parts, axis=0 if mode == "real" else 1)
        got["preview"] = mesh.preview(Nmesh=M, axes=(0, 2))
        if rank == 0:
            one = ArrayMesh(a, BoxSize=64., comm=SelfComm())
            want = {mode: one.compute(mode=mode, Nmesh=M).numpy() for mode in ("real", "complex")}
            want["preview"] = one.preview(Nmesh=M, axes=(0, 2))
            good = all(got[k].shape == want[k].shape and np.allclose(got[k], want[k], rtol=0, atol=1e-12 * np.abs(want[k]).max())
                       for k in want)
            print("resample %d -> %d on %d GPUs: %s" % (Ns, M, world, "OK" if good else "MISMATCH"), flush=True)
            ok &= good
    dist.barrier()
    dist.destroy_process_group()
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
