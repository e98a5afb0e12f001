"""
HOD population benchmark: HaloCatalog.populate / repopulate with the Zheng07, Leauthaud11 or Hearin15 model.

  python bench_hod.py [--model zheng07|leauthaud11|hearin15] [--n 1e7] [--oracle-n 1e6] [--reps 3] [--warmup 1]
                      [--no-chain]

Prints one JSON line: the card and its power limit (read in the same run), and per workload the per-stage CUDA-event
times (hod_occupy, hod_scan, hod_emit, and for Hearin15 hod_percentile, the ranking of the halos in their mass bins that
populate does once and repopulate reuses; mean of --reps runs after --warmup), the bytes the algorithm has to move, the
rate over the stage times and its share of the 3.35 TB/s data-sheet HBM3 bandwidth of the H100 SXM.  Workloads:
  populate      --n halos, dn/dM ~ M^-1.9 over 1e11 - 10^15.5 M_sun/h, uniform in a 2000 Mpc/h box (float32 columns)
  repopulate    the same halos, drawn again in place with another seed
  sat_heavy     repopulate with logM1 = 12.5 (Zheng07) or bsat = 1 (Leauthaud11, Hearin15): many satellites, large
                means through PTRS and the binary-search emit
  chain         LogNormalCatalog(nbar=3e-3, BoxSize=1024, Nmesh=512) -> FOF(0.2, nmin=20) -> to_halos -> populate ->
                FFTPower(Nmesh=512), the wall time of each stage
  oracle        the NumPy oracle at --oracle-n halos, and whether the GPU catalogue of the same halos equals it
Bytes (the percentile stage is not counted): occupy reads the mass and writes two counts (24 B / halo; Hearin15 also
reads the percentile, not counted either); the scan reads and writes the counts (32 B / halo);
emit reads the offsets it searches (counted once, 16 B / halo), the halo columns of its galaxy (3 * 8 + 2 * 12 B) and
writes the galaxy row (3 * 12 + 8 + 4 + 8 B), per galaxy.
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

HBM_BYTES_PER_S = 3.35e12     # NVIDIA H100 SXM data sheet
STAGES = ("hod_occupy", "hod_scan", "hod_emit")
MODELS = ("zheng07", "leauthaud11", "hearin15")
SAT_HEAVY = {"zheng07": dict(logM1=12.5), "leauthaud11": dict(bsat=1.0), "hearin15": dict(bsat=1.0)}


def _model(name):
    from nbodykit_b200.lab import Hearin15Model, Leauthaud11Model, Zheng07Model
    return {"zheng07": Zheng07Model, "leauthaud11": Leauthaud11Model, "hearin15": Hearin15Model}[name]


def _card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = out.stdout.strip() or "not read"
    except Exception:      # noqa: BLE001
        power = "not read"
    return name, power


def _halos(n, seed=1, box=2000.):
    """masses with dn/dM ~ M^-1.9 over [1e11, 10^15.5] by inversion, uniform positions, N(0, 300 km/s) velocities"""
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200.lab import ArrayCatalog, HaloCatalog
    g = torch.Generator(device="cuda").manual_seed(seed)
    u = torch.rand(n, generator=g, device="cuda", dtype=torch.float64)
    a, b, p = 1e11, 10 ** 15.5, -0.9
    mass = (a ** p + u * (b ** p - a ** p)) ** (1 / p)
    pos = torch.rand((n, 3), generator=g, device="cuda", dtype=torch.float32) * box
    vel = torch.randn((n, 3), generator=g, device="cuda", dtype=torch.float32) * 300.
    src = ArrayCatalog({"Mass": mass, "Position": pos, "Velocity": vel}, comm=SelfComm(), BoxSize=box)
    return HaloCatalog(src, Planck15, 0.55)


def _bytes(n, ngal):
    return 24 * n + 32 * n + 16 * n + ngal * (3 * 8 + 2 * 12 + 3 * 12 + 8 + 4 + 8)


def _timed(fn, reps, warmup, stages=STAGES):
    from nbodykit_b200 import _lib
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    _lib.profiler.start()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) / reps
    prof = _lib.profiler.stop()
    st = {k: sum(prof.get(k, [0.0])) / reps for k in stages}
    return wall * 1e3, st


def _entry(wall, st, n, ngal):
    t = sum(v for k, v in st.items() if k in STAGES) * 1e-3
    by = _bytes(n, ngal)
    return dict(halos=n, galaxies=ngal, wall_ms=round(wall, 3), stage_ms={k: round(v, 4) for k, v in st.items()},
                bytes=by, bytes_per_s=by / t if t > 0 else None, share_of_hbm=by / t / HBM_BYTES_PER_S if t > 0 else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=float, default=1e7)
    ap.add_argument("--oracle-n", type=float, default=1e6)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--no-chain", action="store_true")
    ap.add_argument("--model", choices=MODELS, default="zheng07")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    Model = _model(args.model)
    stages = STAGES + (("hod_percentile",) if args.model == "hearin15" else ())
    name, power = _card()
    n = int(args.n)
    res = dict(metric="hod", card=name, power_limit=power, hbm_data_sheet_bytes_per_s=HBM_BYTES_PER_S, workloads={})
    if args.model != "zheng07":
        res["model"] = args.model
    halos = _halos(n)
    box = {}

    def populate():
        box['cat'] = halos.populate(Model, seed=1)
    wall, st = _timed(populate, args.reps, args.warmup, stages)
    cat = box['cat']
    res["workloads"]["populate"] = _entry(wall, st, n, cat.csize)
    wall, st = _timed(lambda: cat.repopulate(seed=2), args.reps, args.warmup, stages)
    res["workloads"]["repopulate"] = _entry(wall, st, n, cat.csize)
    wall, st = _timed(lambda: cat.repopulate(seed=3, **SAT_HEAVY[args.model]), args.reps, args.warmup, stages)
    res["workloads"]["sat_heavy"] = dict(_entry(wall, st, n, cat.csize), fsat=cat.attrs["fsat"])
    del cat, box['cat'], halos
    torch.cuda.empty_cache()

    if not args.no_chain:
        from nbodykit_b200.comm import SelfComm
        from nbodykit_b200.cosmology import NoWiggleEHPower, Planck15
        from nbodykit_b200.lab import FFTPower, FOF, LogNormalCatalog
        chain = {}

        def tick(label, fn):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn()
            torch.cuda.synchronize()
            chain[label] = round((time.perf_counter() - t0) * 1e3, 2)
            return out
        for rep in range(2):       # the first pass warms up every kernel and plan
            src = tick("lognormal", lambda: LogNormalCatalog(Plin=NoWiggleEHPower(redshift=0.55), nbar=3e-3, BoxSize=1024.,
                                                             Nmesh=512, seed=42, comm=SelfComm()))
            fof = tick("fof", lambda: FOF(src, 0.2, nmin=20))
            hc = tick("to_halos", lambda: fof.to_halos(1e12, Planck15, 0.55))
            gal = tick("populate", lambda: hc.populate(Model, seed=42))
            tick("fftpower", lambda: FFTPower(gal, mode="1d", Nmesh=512))
        chain.update(particles=src.csize, halos=hc.csize, galaxies=gal.csize)
        res["workloads"]["chain"] = chain
        del src, fof, hc, gal
        torch.cuda.empty_cache()

    from oracle import hod_models_oracle as hm
    from oracle import hod_oracle as ho
    no = int(args.oracle_n)
    h = _halos(no, seed=5, box=1000.)
    cols = {k: h[k].compute() for k in ("Mass", "Radius", "Concentration", "Position", "Velocity")}
    cols = {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)) for k, v in cols.items()}
    model = Model()
    params = dict(model.param_dict)
    rsd = (1 + 0.55) / (100. * h.cosmo.efunc(0.55))
    t0 = time.perf_counter()
    if args.model == "zheng07":
        want = ho.populate(cols["Mass"], cols["Radius"], cols["Concentration"], cols["Position"], cols["Velocity"],
                           1000., params, 9, rsd=rsd)
    else:
        pct = hm.percentiles(cols["Mass"], cols["Concentration"], model.dlog10_prim_haloprop) \
            if args.model == "hearin15" else None
        want = hm.populate(cols["Mass"], cols["Radius"], cols["Concentration"], cols["Position"], cols["Velocity"],
                           1000., params, 9, 0.55, rsd=rsd, pct=pct, split=getattr(model, "split", 0.5))
    t_or = time.perf_counter() - t0
    got = h.populate(Model, seed=9)
    same_rows = bool(np.array_equal(got["halo_id"].compute().cpu().numpy(), want["halo_id"]))
    gp = got["Position"].compute().cpu().numpy().astype("f8")
    dpos = float(np.abs(gp - want["Position"].astype("f8")).max()) if same_rows else None
    res["workloads"]["oracle"] = dict(halos=no, galaxies=int(want["halo_id"].size), seconds=round(t_or, 3),
                                      same_rows=same_rows, max_abs_position_difference=dpos)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
