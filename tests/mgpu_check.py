"""
Multi-GPU parity check, run under torchrun (one rank per GPU):
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 tests/mgpu_check.py
Every rank holds a share of the particles; the distributed FFTPower (x-slab paint with ghost routing, all-to-all
FFT, all-reduced histogram) must equal the single-GPU result computed on rank 0 from the gathered particles:
mode counts bit-exact, P(k) to 2e-8 (f8) -- and, for the fixed-point tiled paint, the real field itself bit-exact.
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
    failures = []
    L, N = 1000., 64
    rng = np.random.RandomState(1234)
    pos_all = rng.uniform(-50, 1050, size=(400000, 3)).astype("f4")      # includes out-of-box particles
    w_all = rng.uniform(0.5, 1.5, size=len(pos_all))
    mine = slice(rank * len(pos_all) // world, (rank + 1) * len(pos_all) // world)

    cases = [dict(resampler="cic", interlaced=False, dtype="f8", mode="1d", kw={}),
             dict(resampler="tsc", interlaced=True, dtype="f4", mode="2d", kw=dict(Nmu=4, poles=[0, 2])),
             dict(resampler="pcs", interlaced=False, dtype="f8", mode="1d", kw={})]
    peer_stage = None
    for tmode, c in [(t, c) for t in ("push", "nccl") for c in cases]:
        # bulk peer copies pipelined with the y pass (default) | pack + NCCL all-to-all + unpack (platforms without
        # symmetric memory)
        if tmode == "nccl":
            os.environ["NBK_FFT_TRANSPOSE"] = "nccl"
        cat = ArrayCatalog({"Position": torch.from_numpy(pos_all[mine]).cuda(), "Weight": torch.from_numpy(w_all[mine]).cuda()},
                           comm=comm, BoxSize=L)
        mesh = cat.to_mesh(Nmesh=N, resampler=c["resampler"], interlaced=c["interlaced"], compensated=True, dtype=c["dtype"])
        r = FFTPower(mesh, mode=c["mode"], **c["kw"])
        real = mesh.compute(mode="real")
        if tmode == "push":
            peer_stage = getattr(mesh.pm, "_stage", "unused")
        slabs = comm.allgather(real.numpy())
        if rank == 0:
            cat1 = ArrayCatalog({"Position": torch.from_numpy(pos_all).cuda(), "Weight": torch.from_numpy(w_all).cuda()},
                                comm=SelfComm(), BoxSize=L)
            mesh1 = cat1.to_mesh(Nmesh=N, resampler=c["resampler"], interlaced=c["interlaced"], compensated=True, dtype=c["dtype"])
            r1 = FFTPower(mesh1, mode=c["mode"], **c["kw"])
            real1 = mesh1.compute(mode="real").numpy()
            full = np.concatenate(slabs, axis=0)
            # the tiled paint accumulates in fixed point with a quantum of 2^-31 max|w| per deposit, the ghost batches
            # go through the f8 REDG path: agreement is a few quanta x sqrt(deposits per cell) (64 per particle for PCS)
            tol = 2e-8 if c["dtype"] == "f8" else 2e-5
            ok = np.array_equal(r.power["modes"], r1.power["modes"])
            ok &= np.allclose(np.nan_to_num(r.power["power"].real), np.nan_to_num(r1.power["power"].real), rtol=tol,
                              atol=tol * np.nanmax(np.abs(r1.power["power"])))
            ok &= np.allclose(np.nan_to_num(r.power["k"]), np.nan_to_num(r1.power["k"]), rtol=1e-12)
            ok &= r.attrs["N1"] == r1.attrs["N1"] and abs(r.attrs["shotnoise"] - r1.attrs["shotnoise"]) < 1e-9 * r1.attrs["shotnoise"]
            fieldtol = 2e-8 if c["dtype"] == "f8" else 3e-5
            ok &= np.allclose(full, real1, rtol=0, atol=fieldtol * np.abs(real1).max())
            if "poles" in c["kw"]:
                ok &= np.allclose(np.nan_to_num(r.poles["power_2"].real), np.nan_to_num(r1.poles["power_2"].real),
                                  rtol=tol, atol=tol * np.nanmax(np.abs(r1.poles["power_0"])))
            bitexact = (not c["interlaced"]) and np.array_equal(full, real1)
            print("case %s [transpose=%s]: %s (real field bit-identical to 1 GPU: %s)" % (c, tmode, "OK" if ok else "MISMATCH", bitexact), flush=True)
            if not ok:
                failures.append(c)
    os.environ.pop("NBK_FFT_TRANSPOSE", None)
    # ---- a dense catalogue on a 256^3 mesh: tiled paint on slabs (ghost tiles, ordered write-back), both orders
    from nbodykit_b200.cosmology import NoWiggleEHPower
    from nbodykit_b200.lab import LinearMesh, LogNormalCatalog
    big = LogNormalCatalog(Plin=NoWiggleEHPower(), nbar=6e6 / 1000. ** 3, BoxSize=1000., Nmesh=128, bias=2.0, seed=5, comm=SelfComm())
    pbig = big['Position'].compute()
    for order in ("generator", "permuted"):
        pp = pbig
        if order == "permuted":
            g = torch.Generator(device=pbig.device); g.manual_seed(9)
            pp = pbig[torch.randperm(pbig.shape[0], device=pbig.device, generator=g)].contiguous()
        lo, hi = rank * pp.shape[0] // world, (rank + 1) * pp.shape[0] // world
        rd = FFTPower(ArrayCatalog({"Position": pp[lo:hi].contiguous()}, comm=comm, BoxSize=1000.), mode="1d", Nmesh=256)
        if rank == 0:
            r1 = FFTPower(ArrayCatalog({"Position": pp}, comm=SelfComm(), BoxSize=1000.), mode="1d", Nmesh=256)
            ok = np.array_equal(rd.power["modes"], r1.power["modes"]) and np.allclose(
                rd.power["power"].real, r1.power["power"].real, rtol=2e-8, atol=2e-8 * np.nanmax(np.abs(r1.power["power"])))
            print("case 256^3 tiled slabs, %s order: %s" % (order, "OK" if ok else "MISMATCH"), flush=True)
            if not ok:
                failures.append("tiled-slabs-" + order)
    # ---- generators: the shares of a P-rank LogNormalCatalog / LinearMesh are the slabs of the single-rank ones
    lnc = LogNormalCatalog(Plin=NoWiggleEHPower(), nbar=2e-4, BoxSize=1000., Nmesh=64, bias=2.0, seed=5, comm=comm)
    parts = comm.allgather(lnc['Position'].compute().cpu().numpy())
    lin = LinearMesh(NoWiggleEHPower(), BoxSize=1000., Nmesh=64, seed=8, comm=comm)
    plin = FFTPower(lin, mode="1d")
    if rank == 0:
        one = LogNormalCatalog(Plin=NoWiggleEHPower(), nbar=2e-4, BoxSize=1000., Nmesh=64, bias=2.0, seed=5, comm=SelfComm())
        ok = np.array_equal(np.concatenate(parts), one['Position'].compute().cpu().numpy()) and lnc.csize == one.csize
        p1 = FFTPower(LinearMesh(NoWiggleEHPower(), BoxSize=1000., Nmesh=64, seed=8, comm=SelfComm()), mode="1d")
        ok &= np.allclose(plin.power["power"].real, p1.power["power"].real, rtol=1e-5, atol=0)
        print("case generators (LogNormalCatalog shares, LinearMesh): %s" % ("OK" if ok else "MISMATCH"), flush=True)
        if not ok:
            failures.append("generators")
    # ---- FFTRecon (distributed paint + readout): the reconstructed mesh equals the single-GPU one
    from nbodykit_b200.lab import FFTRecon
    rng2 = np.random.RandomState(77)
    centres = rng2.uniform(0, L, size=(200, 3))
    dat = ((centres[rng2.randint(0, 200, size=120000)] + rng2.standard_normal((120000, 3)) * 25.0) % L).astype("f4")
    ran = rng2.uniform(0, L, size=(240000, 3)).astype("f4")
    sl_d = slice(rank * len(dat) // world, (rank + 1) * len(dat) // world)
    sl_r = slice(rank * len(ran) // world, (rank + 1) * len(ran) // world)
    dcat = ArrayCatalog({"Position": torch.from_numpy(dat[sl_d]).cuda()}, comm=comm, BoxSize=L)
    rcat = ArrayCatalog({"Position": torch.from_numpy(ran[sl_r]).cuda()}, comm=comm, BoxSize=L)
    rec = FFTRecon(data=dcat, ran=rcat, Nmesh=N, bias=1.4, f=0.3, R=40., scheme="LF2").compute(mode="real")
    slabs = comm.allgather(rec.numpy())
    if rank == 0:
        one = SelfComm()
        d1 = ArrayCatalog({"Position": torch.from_numpy(dat).cuda()}, comm=one, BoxSize=L)
        r1 = ArrayCatalog({"Position": torch.from_numpy(ran).cuda()}, comm=one, BoxSize=L)
        ref = FFTRecon(data=d1, ran=r1, Nmesh=N, bias=1.4, f=0.3, R=40., scheme="LF2").compute(mode="real").numpy()
        full = np.concatenate(slabs, axis=0)
        ok = np.abs(full - ref).max() <= 1e-4 * np.abs(ref).max()
        print("case FFTRecon LF2: %s (max |diff| / max |field| = %.2e)" % ("OK" if ok else "MISMATCH",
              np.abs(full - ref).max() / np.abs(ref).max()), flush=True)
        if not ok:
            failures.append("FFTRecon")
    if rank == 0:
        st = peer_stage
        print("slab transpose path of the push leg: %s" % ("NVLink peer-memory push" if st not in (None, "unused") else "NCCL all-to-all (%s)" % str(st)), flush=True)
    flag = torch.tensor([len(failures)], device="cuda")
    dist.broadcast(flag, 0)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(1 if int(flag.item()) else 0)


if __name__ == "__main__":
    main()
