"""The x pass of the r2c fused with the FFTPower 1d binning against the two launches it replaces, on one GPU.

    python tools/xbin_bench.py                  # 512^3 and 1024^3, f8
    python tools/xbin_bench.py 1024:f4          # N:dtype (cubic mesh); f4 fields time the separate launches only

For each case the same z + y output (nbk_fft_zy_forward of a random real field) is handed to "separate" --
nbk_fft_lines over x (scaled) followed by nbk_power_bin as FFTPower mode '1d' calls it (CIC compensation, dk = 2 pi / L)
-- and to "fused" -- nbk_fft_x_power_bin, which takes f8 fields only (f4 cases report the separate time alone).
Both are timed with CUDA events after warm-up, median of --reps calls; the separate x pass works in place, so its input
is restored before each call, outside the timed window.  The card's name, power limit and max SM clock are printed with
the numbers.
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nbodykit_b200 import _lib  # noqa: E402
from fftbench import _card  # noqa: E402

DEFAULT = ["512:f8", "1024:f8"]
COMP_CIC = 4       # CompensateCICShotnoise, what a non-interlaced CIC mesh defers to the binning


def _median_ms(fn, before, warmup, reps):
    for _ in range(warmup):
        before()
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        before()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def run_case(spec, warmup, reps, card):
    n, dt = spec.split(":")
    N = int(n)
    code = 4 if dt == "f4" else 8
    tdt = torch.float32 if dt == "f4" else torch.float64
    Nzc = N // 2 + 1
    L = _lib.lib()
    box = 1000.
    real = torch.rand((N, N, N), dtype=tdt, device="cuda")
    zy = torch.empty((N, N, Nzc, 2), dtype=tdt, device="cuda")
    nm = _lib.iarr([N, N, N])
    bx = _lib.darr([box] * 3)
    _lib.check(L.nbk_fft_zy_forward(ctypes.c_void_p(real.data_ptr()), ctypes.c_void_p(zy.data_ptr()), code, N, N, N,
                                    None))
    del real
    work = torch.empty_like(zy)
    dk = 2 * np.pi / box
    kedges = np.arange(0., np.pi * N / box + dk / 2, dk)
    Nx = len(kedges) - 1
    nb = (Nx + 2) * 3
    k2 = _lib.darr((kedges ** 2).astype('f8'))
    mu = _lib.darr([-1., 1.])
    los = _lib.darr([0., 0., 1.])
    vol = box ** 3
    nsum = torch.zeros(nb, dtype=torch.int64, device="cuda")
    facc = torch.zeros(4 * nb, dtype=torch.float64, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    flag = ctypes.c_int(0)

    def zero():
        nsum.zero_()
        facc.zero_()

    def restore():
        zero()
        work.copy_(zy)

    def separate():
        _lib.check(L.nbk_fft_lines(p(work), code, N, N * Nzc, N * Nzc, 1, 0, 0, 1.0 / N ** 3, None))
        _lib.check(L.nbk_power_bin(p(work), None, code, 0, vol, 1, nm, bx, 0, 0, N, 4, k2, Nx, mu, 1, los,
                                   _lib.i32arr([0]), 1, 1, COMP_CIC, COMP_CIC, 0, None, p(nsum), p(facc[:nb]), None,
                                   p(facc[2 * nb:]), None))

    def fused():
        _lib.check(L.nbk_fft_x_power_bin(p(zy), code, nm, bx, 1.0, vol, k2, Nx, mu, 1, los, COMP_CIC, p(nsum),
                                         p(facc[:nb]), p(facc[2 * nb:]), ctypes.byref(flag), None))

    res = dict(N=N, dtype=dt, k_bins=Nx)
    res["separate_ms"] = round(_median_ms(separate, restore, warmup, reps), 4)
    n_sep, f_sep = nsum.cpu().numpy(), facc.cpu().numpy()
    if dt == "f4":
        res.update(card)
        print(json.dumps(res), flush=True)
        return
    res["fused_ms"] = round(_median_ms(fused, zero, warmup, reps), 4)
    if flag.value != 1:
        raise SystemExit("nbk_fft_x_power_bin did not take the fused kernel at N = %d %s" % (N, dt))
    n_fus, f_fus = nsum.cpu().numpy(), facc.cpu().numpy()
    res["fused_over_separate"] = round(res["fused_ms"] / res["separate_ms"], 3)
    res["modes_equal"] = bool(np.array_equal(n_sep, n_fus))
    with np.errstate(invalid='ignore', divide='ignore'):
        rel = np.abs(f_fus - f_sep) / np.abs(f_sep)
    res["max_rel_diff_sums"] = float(np.nanmax(np.where(f_sep != 0, rel, 0.)))
    res["field_gb"] = round(zy.numel() * zy.element_size() / 1e9, 3)
    res.update(card)
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("cases", nargs="*", default=DEFAULT, help="N:dtype")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("xbin_bench needs a CUDA device")
    torch.cuda.set_device(0)
    card = _card()
    for spec in args.cases:
        run_case(spec, args.warmup, args.reps, card)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
