"""Whole-mesh r2c / c2r timing on one GPU, one JSON line per case.

    python tools/fftbench.py                          # the default case list below
    python tools/fftbench.py 96:f8 768:f4:r2c         # side:dtype[:r2c] -- ':r2c' skips the c2r (it needs a third field)

Every case is timed with CUDA events after warm-up (median of --reps calls).  Effective bandwidth counts 6x the real
field's bytes per transform (three passes, each one read and one write of a field of about that size) and is compared
with the 3.35 TB/s HBM3 data-sheet figure of the H100 SXM.  The three passes of the r2c (z, y, x) are also timed one by
one: for power-of-two sides the z pass, the y lines, the x lines and "zy", the z and y passes as the r2c runs them (one
pipelined kernel where it applies); otherwise the mixed-radix passes, and the Bluestein ones on axes whose side has a
prime factor above 7.  The card's name and power limit are printed with the numbers.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nbodykit_b200 import _lib  # noqa: E402
from nbodykit_b200.comm import SelfComm  # noqa: E402
from nbodykit_b200.pmesh.pm import ComplexField, ParticleMesh, RealField  # noqa: E402

DEFAULT = ["512:f8", "768:f8", "1000:f8", "1024:f8", "1536:f4", "1536:f8:r2c"]
HBM_PEAK = 3.35e12


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        power, clock = [s.strip() for s in q[torch.cuda.current_device()].split(",")]
    except Exception:       # noqa: BLE001  (no nvidia-smi: the numbers still stand, the power limit is unknown)
        power, clock = "unknown", "unknown"
    return dict(gpu=torch.cuda.get_device_name(), power_limit=power, max_sm_clock=clock)


def _time(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def _passes(pm, r, c, warmup, reps):
    """ms of the z pass, the y lines and the x lines of the r2c, each the pass ParticleMesh picks for its axis"""
    L = _lib.lib()
    code = 4 if pm.typestr == "f4" else 8
    Nx, Ny, Nz = [int(v) for v in pm.Nmesh]
    Nzc = Nz // 2 + 1
    rp, cp = ctypes.c_void_p(r.value.data_ptr()), ctypes.c_void_p(c.value.data_ptr())
    out = {}
    if pm.pow2:
        # the z pass, the y lines and the x lines one by one, and "zy": the z and y passes as the r2c runs them
        # (nbk_fft_zy_forward: one pipelined kernel where it applies)
        out["z"] = _time(lambda: _lib.check(L.nbk_fft_z_forward(rp, cp, code, Nx * Ny, Nz, None)), warmup, reps)
        out["y"] = _time(lambda: _lib.check(L.nbk_fft_lines(cp, code, Ny, Nzc, Nzc, Nx, Ny * Nzc, 0, 1.0, None)), warmup, reps)
        out["x"] = _time(lambda: _lib.check(L.nbk_fft_lines(cp, code, Nx, Ny * Nzc, Ny * Nzc, 1, 0, 0, 1.0, None)), warmup, reps)
        out["zy"] = _time(lambda: _lib.check(L.nbk_fft_zy_forward(rp, cp, code, Nx, Ny, Nz, None)), warmup, reps)
        return {k: round(v, 3) for k, v in out.items()}
    zp, yp, xp = pm._z_pass(), pm._line_pass(1), pm._line_pass(0)
    out["z"] = _time(lambda: _lib.check(zp(rp, cp, code, Nx * Ny, Nz, 0, 1.0, None)), warmup, reps)
    out["y"] = _time(lambda: _lib.check(yp(cp, cp, code, Ny, Nzc, Nzc, Nx, Ny * Nzc, 0, 1.0, None)), warmup, reps)
    out["x"] = _time(lambda: _lib.check(xp(cp, cp, code, Nx, Ny * Nzc, Ny * Nzc, 1, 0, 0, 1.0, None)), warmup, reps)
    return {k: round(v, 3) for k, v in out.items()}


def run_case(spec, warmup, reps, card):
    parts = spec.split(":")
    n, dtype = int(parts[0]), parts[1]
    with_c2r = not (len(parts) > 2 and parts[2] == "r2c")
    pm = ParticleMesh(BoxSize=1.0, Nmesh=n, dtype=dtype, comm=SelfComm())
    r = RealField(pm)
    r.value.normal_()
    c = ComplexField(pm)
    field_bytes = r.value.numel() * r.value.element_size()
    path = "power-of-two" if pm.pow2 else ("bluestein" if any(pm.bluestein) else "mixed-radix")
    res = dict(case="r2c+c2r" if with_c2r else "r2c", Nmesh=n, dtype=dtype, path=path)
    ms = _time(lambda: r.r2c(out=c), warmup, reps)
    res["r2c_ms"] = round(ms, 3)
    res["r2c_ns_per_cell"] = round(ms * 1e6 / n ** 3, 4)
    res["r2c_GBps"] = round(6 * field_bytes / (ms * 1e-3) / 1e9, 1)
    res["r2c_frac_hbm_peak"] = round(6 * field_bytes / (ms * 1e-3) / HBM_PEAK, 3)
    res["r2c_passes_ms"] = _passes(pm, r, c, warmup, reps)
    if with_c2r:
        ms = _time(lambda: c.c2r(out=r), warmup, reps)
        res["c2r_ms"] = round(ms, 3)
        res["c2r_ns_per_cell"] = round(ms * 1e6 / n ** 3, 4)
        res["c2r_GBps"] = round(6 * field_bytes / (ms * 1e-3) / 1e9, 1)
        res["c2r_frac_hbm_peak"] = round(6 * field_bytes / (ms * 1e-3) / HBM_PEAK, 3)
    res.update(card)
    print(json.dumps(res), flush=True)
    del r, c
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("cases", nargs="*", default=DEFAULT, help="side:dtype[:r2c] (default: %s)" % " ".join(DEFAULT))
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fftbench needs a CUDA device")
    torch.cuda.set_device(0)
    card = _card()
    for spec in args.cases:
        run_case(spec, args.warmup, args.reps, card)


if __name__ == "__main__":
    main()
