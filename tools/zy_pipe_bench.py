"""Forward z + y passes of the power-of-two r2c on one GPU: the pipelined kernel against the two passes it replaces.

    python tools/zy_pipe_bench.py                    # the default cases below
    python tools/zy_pipe_bench.py 4:1024:1024        # x_n:Ny:Nz (f8)

For each case, "pipe" times nbk_fft_zy_forward (k_fft_zy_r2c_pipe where it applies) and "two_pass" times
nbk_fft_z_forward followed by nbk_fft_lines over y, the launches nbk_fft_zy_forward made before the pipelined kernel.
Both are timed with CUDA events after warm-up, median of --reps calls.  Cases cover every (Ny, Nz) shape the kernel
takes at 256 planes and thin slabs of 1 to 16 planes, as the P > 1 slab path runs them.  The card's name, power limit
and max SM clock are printed with the numbers.
"""
import argparse
import ctypes
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nbodykit_b200 import _lib  # noqa: E402
from fftbench import _card, _time  # noqa: E402

SIDES = (256, 512, 1024)
DEFAULT = (["256:%d:%d" % (ny, nz) for ny in SIDES for nz in SIDES] +
           ["%d:1024:1024" % x for x in (1, 2, 4, 8, 16)] + ["%d:512:512" % x for x in (1, 2, 4)])


def run_case(spec, warmup, reps, card):
    x_n, Ny, Nz = [int(v) for v in spec.split(":")]
    Nzc = Nz // 2 + 1
    L = _lib.lib()
    real = torch.randn((x_n, Ny, Nz), dtype=torch.float64, device="cuda")
    cplx = torch.empty((x_n, Ny, Nzc, 2), dtype=torch.float64, device="cuda")
    rp, cp = ctypes.c_void_p(real.data_ptr()), ctypes.c_void_p(cplx.data_ptr())

    def two_pass():
        _lib.check(L.nbk_fft_z_forward(rp, cp, 8, x_n * Ny, Nz, None))
        _lib.check(L.nbk_fft_lines(cp, 8, Ny, Nzc, Nzc, x_n, Ny * Nzc, 0, 1.0, None))

    res = dict(x_n=x_n, Ny=Ny, Nz=Nz, dtype="f8")
    res["pipe_ms"] = round(_time(lambda: _lib.check(L.nbk_fft_zy_forward(rp, cp, 8, x_n, Ny, Nz, None)), warmup, reps), 4)
    res["two_pass_ms"] = round(_time(two_pass, warmup, reps), 4)
    res["pipe_over_two_pass"] = round(res["pipe_ms"] / res["two_pass_ms"], 3)
    res.update(card)
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("cases", nargs="*", default=DEFAULT, help="x_n:Ny:Nz")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("zy_pipe_bench needs a CUDA device")
    torch.cuda.set_device(0)
    card = _card()
    for spec in args.cases:
        run_case(spec, args.warmup, args.reps, card)


if __name__ == "__main__":
    main()
