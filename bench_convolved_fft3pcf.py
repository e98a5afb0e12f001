"""
Survey 3PCF benchmark: ConvolvedFFT3PCF on bench_convolved_bispectrum.py's catalogues (1e7 log-normal objects,
L = 1000 Mpc/h, uniform randoms at 10x the density, constant NZ), both cut to a ball of radius 500 Mpc/h, edges
linspace(0, 150, 9), l = 0 .. 10, CIC, on a 256^3 f8 and a 512^3 f4 mesh of side 1000 * 256 / 210 Mpc/h (about 1219:
the smallest box of a 210^3 / 420^3-compatible cell that passes the geometry guard).

  python bench_convolved_fft3pcf.py [--meshes 256:f8,512:f4] [--warmup 1] [--gram-reps 20]

Prints one JSON line: the card and its power limit (read in the same run); per mesh the wall time of one call after
the warm-up, the CUDA-event stage sums (paint, fill, r2c, product, c2r, gram, all-reduce, ...), the transforms and the
transform time per transform, the listed-tile fraction, the peak device memory; the tile-listed Gram against the dense
Gram on the call's own weight fields (CUDA events over repeated calls); and, reported without a tolerance, the
edge-corrected zeta_0 and zeta_2 of the ball next to FFT3PCF's zeta / mean(F)^3 of the full periodic box on an
uncompensated mesh of the same cell size.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

EDGES = np.linspace(0, 150, 9)
POLES = list(range(11))
RADIUS = 500.
# the survey mesh's cell equals that of a 210^3 (256^3 mesh) or 420^3 (512^3 mesh) mesh of the 1000 Mpc/h box
SURVEY_BOX = 1000. * 256 / 210


def _events(fn, reps):
    """milliseconds per call of fn over `reps` calls, by CUDA events (after one warm call)"""
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def _catalogue():
    from bench_convolved_bispectrum import BOX, N_OBJECTS, SHIFT, _fkp
    fkp = _fkp(N_OBJECTS, BOX)
    ctr = SHIFT + BOX / 2
    c = torch.tensor(ctr, dtype=torch.float64, device="cuda")
    for name in ("data", "randoms"):
        cat = fkp[name]
        p = torch.as_tensor(cat["Position"].compute(), device="cuda")
        cat["Selection"] = ((p.double() - c) ** 2).sum(1) < RADIUS ** 2
    return fkp, ctr


def listed_vs_dense(r, nb, reps):
    """the tile-listed Gram and the dense Gram with the call's weight fields (N and Rf) and nb random bin fields: ms
    per call each and their agreement"""
    from nbodykit_b200 import _lib
    from nbodykit_b200.algorithms.fft3pcf import GRAM_TILE, tile_list
    from nbodykit_b200.pmesh.pm import _CODE, _stream
    mesh = r.first
    D = mesh["data"].to_real_field(normalize=False)
    R = mesh["randoms"].to_real_field(normalize=False)
    D.axpy(R, -r.attrs["alpha"])
    res = []
    L = _lib.lib()
    for name, w in (("N", D), ("Rf", R)):
        pm = w.pm
        code = _CODE[pm.typestr]
        ncell = int(np.prod(pm.real_shape))
        tiles = tile_list(w)
        g = torch.Generator(device="cuda").manual_seed(3)
        store = torch.randn((nb, ncell), dtype=w.value.dtype, device="cuda", generator=g)
        out_l = torch.zeros((nb, nb), dtype=torch.float64, device="cuda")
        out_d = torch.zeros((nb, nb), dtype=torch.float64, device="cuda")

        def listed():
            _lib.check(L.nbk_fft3pcf_gram_tiles(w.value.data_ptr(), store.data_ptr(), ncell, nb, store.data_ptr(), ncell,
                                                nb, code, ncell, tiles.data_ptr(), tiles.numel(), out_l.data_ptr(),
                                                _stream()), "nbk_fft3pcf_gram_tiles")

        def dense():
            _lib.check(L.nbk_fft3pcf_gram(w.value.data_ptr(), store.data_ptr(), ncell, nb, store.data_ptr(), ncell, nb,
                                          code, ncell, out_d.data_ptr(), _stream()), "nbk_fft3pcf_gram")
        # alternated, twice each
        tl, td = [], []
        for _ in range(2):
            tl.append(_events(listed, reps))
            td.append(_events(dense, reps))
        out_l.zero_()
        out_d.zero_()
        listed()
        dense()
        torch.cuda.synchronize()
        a, b = out_l.cpu().numpy(), out_d.cpu().numpy()
        res.append(dict(weight=name, fields=nb, tiles=round(tiles.numel() / -(-ncell // GRAM_TILE), 4),
                        listed_ms=[round(t, 4) for t in tl], dense_ms=[round(t, 4) for t in td],
                        speedup=round(min(td) / min(tl), 3),
                        max_diff_over_max=float(np.max(np.abs(a - b)) / np.max(np.abs(b)))))
        del store
    return res


def periodic_reference(fkp, N, dtype):
    """FFT3PCF's zeta_0, zeta_2 / mean(F)^3 of the full 1000 Mpc/h box of the data (every object, not only the ball)
    at the survey mesh's cell size (uncompensated CIC)"""
    from bench_convolved_bispectrum import BOX, SHIFT
    from nbodykit_b200.lab import ArrayCatalog, FFT3PCF
    pos = torch.as_tensor(fkp["data"]["Position"].compute(), device="cuda")
    d = ArrayCatalog({"Position": pos - torch.as_tensor(SHIFT, dtype=pos.dtype, device=pos.device)}, BoxSize=BOX)
    Np = int(round(N * BOX / SURVEY_BOX))
    mesh = d.to_mesh(Nmesh=Np, BoxSize=BOX, dtype=dtype, resampler="cic", compensated=False)
    mean = float(mesh.compute(mode="real").csum()) / Np ** 3
    r = FFT3PCF(mesh, [0, 2], EDGES)
    return dict(Nmesh=Np, mean=mean, zeta_0=(r.poles["zeta_0"] / mean ** 3).tolist(),
                zeta_2=(r.poles["zeta_2"] / mean ** 3).tolist())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--meshes", default="256:f8,512:f4")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--gram-reps", type=int, default=20)
    args = ap.parse_args()

    from bench_convolved_bispectrum import _card
    from nbodykit_b200 import _lib
    from nbodykit_b200.lab import ConvolvedFFT3PCF
    torch.cuda.set_device(0)
    name, power = _card()
    fkp, ctr = _catalogue()
    res = dict(metric="convolved_fft3pcf", gpus=1, card=name, power_limit=power, radius=RADIUS, box=SURVEY_BOX,
               edges=EDGES.tolist(), poles=POLES, resampler="cic",
               selected={s: int(torch.as_tensor(fkp[s]["Selection"].compute()).sum().item()) for s in ("data", "randoms")}, meshes={})
    for spec in args.meshes.split(","):
        N, dtype = spec.split(":")
        N = int(N)
        mesh = fkp.to_mesh(Nmesh=N, BoxSize=SURVEY_BOX, BoxCenter=ctr, dtype=dtype, resampler="cic")
        for _ in range(args.warmup):
            ConvolvedFFT3PCF(mesh, POLES, EDGES)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        _lib.profiler.start()
        t0 = time.perf_counter()
        r = ConvolvedFFT3PCF(mesh, POLES, EDGES)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        stages = {k: round(sum(v), 3) for k, v in _lib.profiler.stop().items()}
        peak = torch.cuda.max_memory_allocated() / 2 ** 30
        nt = int(r.attrs["transforms"])
        tr_ms = stages.get("fft3pcf_r2c", 0.) + stages.get("fft3pcf_c2r", 0.)
        res["meshes"]["%d^3 %s" % (N, dtype)] = dict(
            seconds=round(wall, 4), stages_ms=stages, transforms=nt, transform_ms_total=round(tr_ms, 3),
            ms_per_transform=round(tr_ms / nt, 4), tiles=round(float(r.attrs["tiles"]), 4),
            peak_mem_gib=round(peak, 3), alpha=r.attrs["alpha"],
            gram_listed_vs_dense=listed_vs_dense(r, 8, args.gram_reps),
            zeta_0=r.poles["zeta_0"].tolist(), zeta_2=r.poles["zeta_2"].tolist(),
            periodic=periodic_reference(fkp, N, dtype))
        del r, mesh
    print(json.dumps(res))


if __name__ == "__main__":
    main()
