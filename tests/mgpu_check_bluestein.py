"""
Multi-GPU parity check of the Bluestein FFT route, run under torchrun (one rank per GPU):
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29521 tests/mgpu_check_bluestein.py
FFTPower at Nmesh = [44, 44, 37] (every side has a prime factor above 7: Bluestein z pass, y and x lines around the NCCL
all-to-all) on P GPUs must equal the single-GPU result computed on rank 0 from the gathered particles: mode counts
bit-exact, P(k) to 2e-8 (f8).
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
    from nbodykit_b200.lab import ArrayCatalog, FFTPower
    comm = CurrentMPIComm.get()
    assert comm.size == world
    N, L, kw = [44, 44, 37], [550., 550., 460.], dict(mode="2d", Nmu=4, poles=[0, 2])
    rng = np.random.RandomState(4321)
    pos_all = (rng.uniform(0, 1, size=(200000, 3)) * np.asarray(L)).astype("f4")
    w_all = rng.uniform(0.5, 1.5, size=len(pos_all))
    mine = slice(rank * len(pos_all) // world, (rank + 1) * len(pos_all) // world)
    cat = ArrayCatalog({"Position": torch.from_numpy(pos_all[mine]).cuda(), "Weight": torch.from_numpy(w_all[mine]).cuda()},
                       comm=comm, BoxSize=L)
    r = FFTPower(cat.to_mesh(Nmesh=N, resampler="cic", compensated=True, dtype="f8"), **kw)
    ok = True
    if rank == 0:
        cat1 = ArrayCatalog({"Position": torch.from_numpy(pos_all).cuda(), "Weight": torch.from_numpy(w_all).cuda()},
                            comm=SelfComm(), BoxSize=L)
        r1 = FFTPower(cat1.to_mesh(Nmesh=N, resampler="cic", compensated=True, dtype="f8"), **kw)
        tol = 2e-8
        ok = np.array_equal(r.power["modes"], r1.power["modes"])
        ok &= np.allclose(np.nan_to_num(r.power["power"].real), np.nan_to_num(r1.power["power"].real), rtol=tol,
                          atol=tol * np.nanmax(np.abs(r1.power["power"])))
        ok &= np.allclose(np.nan_to_num(r.power["k"]), np.nan_to_num(r1.power["k"]), rtol=1e-12)
        ok &= np.allclose(np.nan_to_num(r.poles["power_2"].real), np.nan_to_num(r1.poles["power_2"].real), rtol=tol,
                          atol=tol * np.nanmax(np.abs(r1.poles["power_0"])))
        print("Nmesh %s on %d GPUs: %s" % (N, world, "OK" if ok else "MISMATCH"), flush=True)
    dist.barrier()
    dist.destroy_process_group()
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
