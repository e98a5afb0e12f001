"""
The forward z + y passes of the power-of-two r2c (nbk_fft_zy_forward) against the two passes they combine: the z pass
(nbk_fft_z_forward) followed by the y lines (nbk_fft_lines).  Where the pipelined kernel runs (f8, Nz and Ny in
{256, 512, 1024}) it must give the same bits; elsewhere nbk_fft_zy_forward runs those two passes itself, so the f4
cases only check that fallback, and so do slabs of at most D planes (the pipeline depth: the y tiles trail the z rows
by D planes), which fit in half the L2.  The plane counts cover one plane, a few, D and D + 1, and many.  Every case calls nbk_fft_zy_forward twice in a row: the second call must see
none of the first call's progress flags.  Calls on two streams may overlap and must not see each other's.
"""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SIDES = [256, 512, 1024]


def _lib():
    from nbodykit_b200 import _lib
    return _lib


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _depth(Ny, Nz, itemsize):
    """planes the y tiles trail the z rows by: the waiting planes and the one being transformed fill half the L2"""
    l2 = torch.cuda.get_device_properties(torch.cuda.current_device()).L2_cache_size
    plane = Ny * (Nz // 2 + 1) * 2 * itemsize
    return max(1, l2 // (2 * plane) - 1)


def _two_passes(real, x_n, Ny, Nz, code):
    L = _lib()
    Nzc = Nz // 2 + 1
    out = torch.empty((x_n, Ny, Nzc, 2), dtype=real.dtype, device=real.device)
    L.check(L.lib().nbk_fft_z_forward(_p(real), _p(out), code, x_n * Ny, Nz, None), "fft_z_forward")
    L.check(L.lib().nbk_fft_lines(_p(out), code, Ny, Nzc, Nzc, x_n, Ny * Nzc, 0, 1.0, None), "fft_lines")
    return out


def _zy(real, x_n, Ny, Nz, code):
    L = _lib()
    out = torch.full((x_n, Ny, Nz // 2 + 1, 2), float("nan"), dtype=real.dtype, device=real.device)
    L.check(L.lib().nbk_fft_zy_forward(_p(real), _p(out), code, x_n, Ny, Nz, None), "fft_zy_forward")
    return out


def _check(x_n, Ny, Nz, dtype):
    torch.cuda.set_device(0)
    tdt = torch.float32 if dtype == "f4" else torch.float64
    code = 4 if dtype == "f4" else 8
    g = torch.Generator(device="cuda").manual_seed(1000 * Ny + Nz + x_n)
    real = torch.randn((x_n, Ny, Nz), dtype=tdt, device="cuda", generator=g)
    ref = _two_passes(real, x_n, Ny, Nz, code)
    for call in range(2):
        got = _zy(real, x_n, Ny, Nz, code)
        torch.cuda.synchronize()
        assert torch.equal(got, ref), "call %d: %s x_n=%d Ny=%d Nz=%d differs from z pass + y lines" % (
            call, dtype, x_n, Ny, Nz)


@pytest.mark.parametrize("dtype", ["f4", "f8"])
@pytest.mark.parametrize("Ny", SIDES)
@pytest.mark.parametrize("Nz", SIDES)
@pytest.mark.parametrize("planes", ["1", "2", "3", "D", "D+1", "5", "64"])
def test_zy_forward_bit_equal_to_two_passes(cuda, dtype, Ny, Nz, planes):
    D = _depth(Ny, Nz, 4 if dtype == "f4" else 8)
    x_n = {"D": D, "D+1": D + 1}.get(planes) or int(planes)
    _check(x_n, Ny, Nz, dtype)


def test_zy_forward_bit_equal_1024_cube_f8(cuda):
    _check(1024, 1024, 1024, "f8")


def test_zy_forward_concurrent_streams(cuda):
    torch.cuda.set_device(0)
    L = _lib()
    x_n, Ny, Nz = 96, 1024, 1024
    g = torch.Generator(device="cuda").manual_seed(11)
    reals = [torch.randn((x_n, Ny, Nz), dtype=torch.float64, device="cuda", generator=g) for _ in range(2)]
    refs = [_two_passes(r, x_n, Ny, Nz, 8) for r in reals]
    outs = [torch.full_like(refs[0], float("nan")) for _ in range(2)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for rep in range(3):
        for r, o, st in zip(reals, outs, streams):
            with torch.cuda.stream(st):
                L.check(L.lib().nbk_fft_zy_forward(_p(r), _p(o), 8, x_n, Ny, Nz, ctypes.c_void_p(st.cuda_stream)),
                        "fft_zy_forward")
        torch.cuda.synchronize()
        for i in range(2):
            assert torch.equal(outs[i], refs[i]), "repeat %d, stream %d differs from z pass + y lines" % (rep, i)
            outs[i].fill_(float("nan"))
        torch.cuda.synchronize()


def test_r2c_256_cube_matches_numpy(cuda):
    torch.cuda.set_device(0)
    L = _lib()
    N = 256
    rng = np.random.RandomState(3)
    x = rng.standard_normal((N, N, N))
    real = torch.from_numpy(x).cuda()
    out = torch.empty((N, N, N // 2 + 1), dtype=torch.complex128, device="cuda")
    nm = (ctypes.c_int64 * 3)(N, N, N)
    for _ in range(2):
        out.zero_()
        L.check(L.lib().nbk_r2c(_p(real), _p(out), 8, nm, 1.0, None), "nbk_r2c")
        got = out.cpu().numpy()
        ref = np.fft.rfftn(x) / N ** 3
        err = np.abs(got - ref).max() / np.abs(ref).max()
        assert err < 1e-13, err
