"""
FFT 3PCF benchmark: FFT3PCF on bench_3pcf.py's boss_like LogNormalCatalog (1e6 objects, L = 2500 Mpc/h), edges
linspace(0, 150, 9), l = 0 .. 10, painted on a 256^3 f8 and a 512^3 f4 mesh; SimulationBox3PCF on the same catalogue in
the same run, for the wall-time comparison only (the two estimators differ by the mesh, so their values are not
compared); and the register-blocked Gram (nbk_fft3pcf_gram) against nbk_bispec_triple_sum on the same fields with the
rows (w, a_i, a_j), i <= j.

  python bench_fft3pcf.py [--meshes 256:f8,512:f4] [--warmup 1] [--gram-reps 20]

Prints one JSON line: the card and its power limit (read in the same run); per mesh the wall time of the call, the
CUDA-event sums per stage (paint, fill, r2c, product, c2r, gram, ...), the transforms run and the transform time per
transform, and the peak device memory; SimulationBox3PCF's wall time; and the Gram against the triple sum.
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


def gram_vs_triple_sum(N, dtype, nb, reps):
    """the Gram and the triple sum on 1 + nb random fields of an N^3 mesh: ms per call each, and their agreement"""
    from nbodykit_b200 import _lib
    from nbodykit_b200.pmesh.pm import _stream
    tdt = torch.float64 if dtype == "f8" else torch.float32
    code = 8 if dtype == "f8" else 4
    ncell = N ** 3
    g = torch.Generator(device="cuda").manual_seed(3)
    store = torch.randn((1 + nb, ncell), dtype=tdt, device="cuda", generator=g)
    iu = np.triu_indices(nb)
    rows = np.stack([np.zeros(len(iu[0]), dtype="i4"), iu[0] + 1, iu[1] + 1], axis=1).astype("i4")
    tri = torch.from_numpy(np.ascontiguousarray(rows)).cuda()
    out_g = torch.zeros((nb, nb), dtype=torch.float64, device="cuda")
    out_t = torch.zeros(len(rows), dtype=torch.float64, device="cuda")
    L = _lib.lib()

    def gram():
        _lib.check(L.nbk_fft3pcf_gram(store[0].data_ptr(), store[1].data_ptr(), ncell, nb, store[1].data_ptr(), ncell, nb,
                                      code, ncell, out_g.data_ptr(), _stream()), "nbk_fft3pcf_gram")

    def triple():
        _lib.check(L.nbk_bispec_triple_sum(store.data_ptr(), code, ncell, 1 + nb, ncell, tri.data_ptr(), len(rows),
                                           out_t.data_ptr(), _stream()), "nbk_bispec_triple_sum")
    tg = _events(gram, reps)
    tt = _events(triple, reps)
    out_g.zero_()
    out_t.zero_()
    gram()
    triple()
    torch.cuda.synchronize()
    a = out_g.cpu().numpy()[iu]
    b = out_t.cpu().numpy()
    rel = float(np.max(np.abs(a - b)) / np.max(np.abs(b)))
    return dict(mesh=N, dtype=dtype, fields=nb, pairs=len(rows), gram_ms=round(tg, 4), triple_sum_ms=round(tt, 4),
                speedup=round(tt / tg, 3), max_diff_over_max=rel)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--meshes", default="256:f8,512:f4")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--gram-reps", type=int, default=20)
    args = ap.parse_args()

    from bench_3pcf import SIZES, _card, _catalog
    from nbodykit_b200 import _lib
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import FFT3PCF, SimulationBox3PCF
    torch.cuda.set_device(0)
    name, power = _card()
    n, L = SIZES["boss_like"]
    src = _catalog(n, L, SelfComm())
    res = dict(metric="fft3pcf", card=name, power_limit=power, objects=int(src.csize), box=L, edges=EDGES.tolist(),
               poles=POLES, meshes={})
    for spec in args.meshes.split(","):
        N, dtype = spec.split(":")
        N = int(N)
        mesh = src.to_mesh(Nmesh=N, BoxSize=L, dtype=dtype, compensated=True)
        for _ in range(args.warmup):
            FFT3PCF(mesh, POLES, EDGES)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        _lib.profiler.start()
        t0 = time.perf_counter()
        r = FFT3PCF(mesh, POLES, EDGES)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        stages = {k.replace("fft3pcf_", ""): round(sum(v), 3) for k, v in _lib.profiler.stop().items()
                  if k.startswith("fft3pcf")}
        nt = int(r.attrs["transforms"])
        tr_ms = stages.get("r2c", 0.) + stages.get("c2r", 0.)
        res["meshes"]["%d^3 %s" % (N, dtype)] = dict(
            seconds=round(wall, 4), stages_ms=stages, transforms=nt, transform_ms_total=round(tr_ms, 3),
            ms_per_transform=round(tr_ms / nt, 4), peak_mem_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 3),
            nsep=[int(v) for v in r.nsep])
        del r, mesh
    # SimulationBox3PCF on the same catalogue: wall time only
    for _ in range(args.warmup):
        SimulationBox3PCF(src, POLES, EDGES)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    SimulationBox3PCF(src, POLES, EDGES)
    torch.cuda.synchronize()
    res["simulationbox3pcf_seconds"] = round(time.perf_counter() - t0, 4)
    del src
    res["gram_vs_triple_sum"] = [gram_vs_triple_sum(256, "f8", 8, args.gram_reps),
                                 gram_vs_triple_sum(512, "f4", 8, args.gram_reps),
                                 gram_vs_triple_sum(256, "f8", 32, args.gram_reps)]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
