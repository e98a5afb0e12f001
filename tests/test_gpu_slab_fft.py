"""
The power-of-two slab transform of P > 1 runs (RealField.r2c / ComplexField.c2r in pmesh/pm.py) on P virtual ranks of
one GPU, against float64 NumPy.

Every rank's slab is its own tensor and is called with the arguments pm.py passes.  The two exchange routes are
driven kernel by kernel:
  * peer route: the "peers" are P staging buffers of this device; forward = z pass, y pass into send blocks in
    _push_chunks(x_n) parts, bulk push, x pass out of place; inverse = x pass into send blocks, push into the staging
    buffer viewed as [x_n][Ny][Nzc], y + z c2r;
  * all-to-all route: pack, a block swap done here (block q of rank r's receive buffer is block r of rank q's send
    buffer), unpack, in-place line pass.
A spectrum with no symmetry has a NumPy c2r as well, irfftn (complex inverses along x and y, a real inverse along z that
drops the imaginary parts of the kz = 0 and kz = Nz/2 entries): both routes and the single-GPU nbk_c2r must equal it.

The peer route needs symmetric memory shared between processes, which one process on one GPU does not have, so these
tests check the kernels with their own copy of the arguments of pm.py's peer branch: an argument error in that branch
itself (x_start / y_start, rows_per_peer, chunk bounds, the staging view) is not seen here.  pm.py's all-to-all branch
runs end to end in tests/test_gpu_slab_route.py.
"""
import ctypes

import numpy as np
import pytest
from gpu_helpers import code as _code, dev as _dev, host as _host, nbk as _lib, ptr as _p

pytestmark = pytest.mark.gpu

# (Nx, Ny, Nz, P): x_n = y_n = 1 (Nx = Ny = P, P up to the 16 peers of the exchange), Nx != Ny, x_n of 1 and 2 (the
# chunked push with fewer parts than 4), lines of every kernel regime (< 64 shared memory, 64 / 128 register I/O,
# 256 / 512 / 1024 TMA, 2048), Nz = 4 (Nzc = 3: the misaligned f4 fallback), Nz = 256 / 512 / 1024 (the TMA z pass)
# and a long z row
SLAB_CASES = [
    (2, 2, 8, 2),
    (4, 4, 4, 4),
    (16, 16, 8, 16),
    (16, 32, 4, 8),
    (8, 64, 16, 4),
    (32, 8, 32, 2),
    (128, 16, 256, 2),
    (16, 256, 512, 4),
    (512, 8, 16, 8),
    (4, 1024, 1024, 4),
    (2048, 4, 8, 4),
    (8, 8, 4096, 2),
    (64, 128, 4, 16),
]
TOL = {"f8": 1e-13, "f4": 2e-6}
SCALE = 2.5          # extra_scale of the forward transform: r2c folds it into the x pass


def _ids(c):
    return "%dx%dx%d-P%d" % c


def _cdt(dtype):
    import torch
    return torch.complex64 if dtype == "f4" else torch.complex128


def _rdt(dtype):
    import torch
    return torch.float32 if dtype == "f4" else torch.float64


def _push_chunks(x_n):
    from nbodykit_b200.pmesh.pm import _push_chunks
    return _push_chunks(x_n)


def _swap(send, P):
    """the all-to-all: rank r receives block r of every rank q's send buffer, in rank order"""
    import torch
    return [torch.cat([send[q].view(P, -1)[r] for q in range(P)]).contiguous() for r in range(P)]


# ---- forward -------------------------------------------------------------------------------------------------------
def forward_peer(slabs, N, P, dtype, scale):
    import torch
    L, ch = _lib(), _lib().check
    Nx, Ny, Nz = N
    x_n, y_n, Nzc = Nx // P, Ny // P, Nz // 2 + 1
    code = _code(dtype)
    stage = [torch.zeros((y_n, Nx, Nzc), dtype=_cdt(dtype), device="cuda") for _ in range(P)]
    ptrs = (ctypes.c_void_p * P)(*[t.data_ptr() for t in stage])
    nchunk = _push_chunks(x_n)
    per = (x_n + nchunk - 1) // nchunk
    for r in range(P):
        work = torch.empty((x_n, Ny, Nzc), dtype=_cdt(dtype), device="cuda")
        send = torch.zeros((P, y_n, x_n, Nzc), dtype=_cdt(dtype), device="cuda")
        ch(L.lib().nbk_fft_z_forward(_p(slabs[r]), _p(work), code, x_n * Ny, Nz, None), "fft_z_forward")
        for c in range(nchunk):
            o0 = c * per
            oc = min(per, x_n - o0)
            if oc <= 0:
                break
            ch(L.lib().nbk_fft_lines_pack_range(_p(work), _p(send), code, Ny, Nzc, x_n, o0, oc, P, 0, 1.0, None),
               "fft_lines_pack_range")
            ch(L.lib().nbk_slab_push_range(_p(send), ptrs, code, y_n, x_n, Nzc, r * x_n, o0, oc, P, r, None),
               "slab_push_range")
    out = []
    s = float(scale) / (float(Nx) * Ny * Nz)
    for r in range(P):
        o = torch.empty_like(stage[r])
        ch(L.lib().nbk_fft_lines_oop(_p(stage[r]), _p(o), code, Nx, Nzc, Nzc, y_n, Nx * Nzc, 0, s, None), "fft_lines_oop")
        out.append(o)
    return out


def forward_nccl(slabs, N, P, dtype, scale):
    import torch
    L, ch = _lib(), _lib().check
    Nx, Ny, Nz = N
    x_n, y_n, Nzc = Nx // P, Ny // P, Nz // 2 + 1
    code = _code(dtype)
    sends = []
    for r in range(P):
        work = torch.empty((x_n, Ny, Nzc), dtype=_cdt(dtype), device="cuda")
        send = torch.empty_like(work)
        ch(L.lib().nbk_fft_zy_forward(_p(slabs[r]), _p(work), code, x_n, Ny, Nz, None), "fft_zy_forward")
        ch(L.lib().nbk_transpose_pack(_p(work), _p(send), code, x_n, Ny, Nzc, P, None), "transpose_pack")
        sends.append(send)
    out = []
    s = float(scale) / (float(Nx) * Ny * Nz)
    for r, recv in enumerate(_swap(sends, P)):
        o = torch.empty((y_n, Nx, Nzc), dtype=_cdt(dtype), device="cuda")
        ch(L.lib().nbk_transpose_unpack(_p(recv), _p(o), code, y_n, Nx, Nzc, P, None), "transpose_unpack")
        ch(L.lib().nbk_fft_lines(_p(o), code, Nx, Nzc, Nzc, y_n, Nx * Nzc, 0, s, None), "fft_lines(x)")
        out.append(o)
    return out


# ---- inverse -------------------------------------------------------------------------------------------------------
def inverse_peer(specs, N, P, dtype):
    import torch
    L, ch = _lib(), _lib().check
    Nx, Ny, Nz = N
    x_n, y_n, Nzc = Nx // P, Ny // P, Nz // 2 + 1
    code = _code(dtype)
    # the staging buffer has the shape of the transposed field; the c2r push fills it as [x_n][Ny][Nzc]
    stage = [torch.zeros((y_n, Nx, Nzc), dtype=_cdt(dtype), device="cuda") for _ in range(P)]
    ptrs = (ctypes.c_void_p * P)(*[t.data_ptr() for t in stage])
    for r in range(P):
        send = torch.zeros((P, x_n, y_n, Nzc), dtype=_cdt(dtype), device="cuda")
        ch(L.lib().nbk_fft_lines_pack_range(_p(specs[r]), _p(send), code, Nx, Nzc, y_n, 0, y_n, P, 1, 1.0, None),
           "fft_lines_pack_range(inverse)")
        ch(L.lib().nbk_slab_push_range(_p(send), ptrs, code, x_n, y_n, Nzc, r * y_n, 0, y_n, P, r, None),
           "slab_push_range(inverse)")
    out = []
    for r in range(P):
        o = torch.empty((x_n, Ny, Nz), dtype=_rdt(dtype), device="cuda")
        ch(L.lib().nbk_fft_zy_backward(_p(stage[r]), _p(o), code, x_n, Ny, Nz, None), "fft_zy_backward")
        out.append(o)
    return out


def inverse_nccl(specs, N, P, dtype):
    import torch
    L, ch = _lib(), _lib().check
    Nx, Ny, Nz = N
    x_n, y_n, Nzc = Nx // P, Ny // P, Nz // 2 + 1
    code = _code(dtype)
    sends = []
    for r in range(P):
        work = specs[r].clone()
        ch(L.lib().nbk_fft_lines(_p(work), code, Nx, Nzc, Nzc, y_n, Nx * Nzc, 1, 1.0, None), "fft_lines(x)")
        send = torch.empty_like(work)
        ch(L.lib().nbk_transpose_pack_back(_p(work), _p(send), code, y_n, Nx, Nzc, P, None), "pack_back")
        sends.append(send)
    out = []
    for r, recv in enumerate(_swap(sends, P)):
        slab = torch.empty((x_n, Ny, Nzc), dtype=_cdt(dtype), device="cuda")
        ch(L.lib().nbk_transpose_unpack_back(_p(recv), _p(slab), code, x_n, Ny, Nzc, P, None), "unpack_back")
        o = torch.empty((x_n, Ny, Nz), dtype=_rdt(dtype), device="cuda")
        ch(L.lib().nbk_fft_zy_backward(_p(slab), _p(o), code, x_n, Ny, Nz, None), "fft_zy_backward")
        out.append(o)
    return out


ROUTES = {"peer": (forward_peer, inverse_peer), "nccl": (forward_nccl, inverse_nccl)}


def _split_x(a, P):
    x_n = a.shape[0] // P
    return [_dev(a[r * x_n:(r + 1) * x_n]) for r in range(P)]


def _split_y(c, P):
    """rank r's transposed y slab [y_n][Nx][Nzc]"""
    y_n = c.shape[1] // P
    return [_dev(c[:, r * y_n:(r + 1) * y_n].transpose(1, 0, 2)) for r in range(P)]


def _join_y(parts):
    return np.concatenate([_host(p).transpose(1, 0, 2) for p in parts], axis=1)


def _join_x(parts):
    return np.concatenate([_host(p) for p in parts], axis=0)


def _spec_err(got, want, dtype, n):
    """max error in units of the test_r2c_c2r tolerance: rms |want| x log2(N^3) x TOL"""
    return np.abs(got - want).max() / (TOL[dtype] * np.sqrt((np.abs(want) ** 2).mean()) * np.log2(n))


def _real_err(got, want, dtype, n):
    """max error in units of the test_r2c_c2r round-trip tolerance (unit-variance fields): 10 log2(N^3) x TOL"""
    return np.abs(got - want).max() / (TOL[dtype] * 10 * np.log2(n))


# ---------------------------------------------------------------------------------------------
# forward and inverse against NumPy, both routes
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", SLAB_CASES, ids=_ids)
@pytest.mark.parametrize("dtype", ["f8", "f4"])
@pytest.mark.parametrize("route", sorted(ROUTES))
def test_slab_r2c_c2r(cuda, case, dtype, route):
    """each rank's [y_n][Nx][Nzc] equals extra_scale rfftn(x) / N^3 transposed; the inverse of the spectrum of a real
    field gives irfftn N^3 on each x slab; forward + inverse returns the input"""
    Nx, Ny, Nz, P = case
    N = (Nx, Ny, Nz)
    n = Nx * Ny * Nz
    fwd, inv = ROUTES[route]
    real = np.random.RandomState(sum(case)).standard_normal(N).astype(dtype)
    want = np.fft.rfftn(real.astype("f8")) * (SCALE / n)
    spec = fwd(_split_x(real, P), N, P, dtype, SCALE)
    got = _join_y(spec)
    assert got.shape == want.shape
    assert _spec_err(got, want, dtype, n) <= 1, "forward %s" % route
    # the inverse of a spectrum given in f8 (cast to the field dtype)
    c = (np.fft.rfftn(real.astype("f8")) / n).astype("c8" if dtype == "f4" else "c16")
    ref = np.fft.irfftn(c.astype("c16"), s=N, axes=(0, 1, 2)) * n
    back = _join_x(inv(_split_y(c, P), N, P, dtype))
    assert _real_err(back, ref, dtype, n) <= 1, "inverse %s" % route
    # the round trip through both distributed passes
    trip = _join_x(inv([s * (1.0 / SCALE) for s in spec], N, P, dtype))
    assert _real_err(trip, real.astype("f8"), dtype, n) <= 1, "round trip %s" % route


@pytest.mark.parametrize("case", SLAB_CASES, ids=_ids)
@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_slab_c2r_general_input_equals_one_gpu(cuda, case, dtype):
    """a spectrum with no symmetry (complex kz = 0 and Nyquist planes included): the single-GPU nbk_c2r equals irfftn
    N^3 of it, and both distributed inverses, which run the same x, y, z passes, agree with nbk_c2r to rounding"""
    import torch
    _l = _lib()
    Nx, Ny, Nz, P = case
    N = (Nx, Ny, Nz)
    n = Nx * Ny * Nz
    rng = np.random.RandomState(7 + sum(case))
    shape = (Nx, Ny, Nz // 2 + 1)
    c = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype("c8" if dtype == "f4" else "c16")
    full = _dev(c)
    one = torch.empty(N, dtype=_rdt(dtype), device="cuda")
    work = torch.empty_like(full)
    _l.check(_l.lib().nbk_c2r(_p(full), _p(one), _code(dtype), _l.iarr(N), _p(work), None), "nbk_c2r")
    want = _host(one).astype("f8")
    np.testing.assert_array_equal(_host(full), c)          # nbk_c2r with `work` keeps its input
    rms = np.sqrt((want ** 2).mean())
    ref = np.fft.irfftn(c.astype("c16"), s=N, axes=(0, 1, 2)) * n
    assert np.abs(want - ref).max() <= TOL[dtype] * rms * np.log2(n) * 10, "nbk_c2r vs irfftn"
    for route, (_, inv) in sorted(ROUTES.items()):
        specs = _split_y(c, P)
        got = _join_x(inv(specs, N, P, dtype))
        err = np.abs(got - want).max()
        assert err <= TOL[dtype] * rms * np.log2(n), "%s: %g vs rms %g" % (route, err, rms)
        assert np.abs(got - ref).max() <= TOL[dtype] * rms * np.log2(n) * 10, "%s vs irfftn" % route
        if route == "peer":                                 # the peer inverse only reads its input
            np.testing.assert_array_equal(_join_y(specs), c)


# ---------------------------------------------------------------------------------------------
# the z + y passes of an x slab alone
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(1, 8, 4), (1, 64, 256), (2, 2, 16), (3, 256, 8), (1, 1024, 32), (5, 16, 1024),
                                   (1, 2048, 4), (2, 4, 4096)])
@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_zy_forward_backward_x_slab(cuda, shape, dtype):
    """nbk_fft_zy_forward: fft_y(rfft_z(x)) unnormalised; nbk_fft_zy_backward: its unnormalised inverse, on x slabs of
    x_n planes (x_n = 1 included)"""
    import torch
    _l = _lib()
    x_n, Ny, Nz = shape
    n = Ny * Nz
    real = np.random.RandomState(x_n * Ny + Nz).standard_normal(shape).astype(dtype)
    want = np.fft.fft(np.fft.rfft(real.astype("f8"), axis=2), axis=1)
    cpl = torch.empty((x_n, Ny, Nz // 2 + 1), dtype=_cdt(dtype), device="cuda")
    _l.check(_l.lib().nbk_fft_zy_forward(_p(_dev(real)), _p(cpl), _code(dtype), x_n, Ny, Nz, None), "fft_zy_forward")
    got = _host(cpl)
    assert _spec_err(got, want, dtype, n) <= 1
    c = want.astype("c8" if dtype == "f4" else "c16")
    ref = np.fft.irfft(np.fft.ifft(c.astype("c16"), axis=1), n=Nz, axis=2) * n
    out = torch.empty(shape, dtype=_rdt(dtype), device="cuda")
    _l.check(_l.lib().nbk_fft_zy_backward(_p(_dev(c)), _p(out), _code(dtype), x_n, Ny, Nz, None), "fft_zy_backward")
    assert np.abs(_host(out) - ref).max() <= TOL[dtype] * np.sqrt(n) * 10 * np.log2(n)


# ---------------------------------------------------------------------------------------------
# the documented line limits, one GPU
# ---------------------------------------------------------------------------------------------
LIMIT_SHAPES = [(4096, 2, 4), (2, 4096, 4), (4, 4096, 8), (2, 2, 8192), (8192, 2, 4), (2, 8192, 4), (2, 2, 16384)]


# (longest x / y line, longest z row) of the power-of-two transform per dtype (check_dims in csrc/fft.cu)
POW2_LIMITS = {"f8": (4096, 8192), "f4": (8192, 16384)}


def _limit_ok(N, dtype):
    lines, nz = POW2_LIMITS[dtype]
    return N[0] <= lines and N[1] <= lines and N[2] <= nz


@pytest.mark.parametrize("N", LIMIT_SHAPES, ids=lambda N: "%dx%dx%d" % N)
@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_pow2_limits_one_gpu(cuda, N, dtype):
    """x / y lines of 4096 and 8192 points and z rows of 8192 and 16384: inside the limits of the dtype r2c equals
    NumPy and c2r inverts it; outside, r2c and c2r raise with a message naming the limit"""
    from nbodykit_b200._lib import NbkError
    from nbodykit_b200.pmesh.pm import RealField, ComplexField
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.pmesh.pm import ParticleMesh
    n = int(np.prod(N))
    pm = ParticleMesh(BoxSize=1.0, Nmesh=N, dtype=dtype, comm=SelfComm())
    real = np.random.RandomState(3).standard_normal(N).astype(dtype)
    f = RealField(pm)
    f[...] = real
    if not _limit_ok(N, dtype):
        with pytest.raises(NbkError, match="at most"):
            f.r2c()
        with pytest.raises(NbkError, match="at most"):
            ComplexField(pm).c2r()
        return
    c = f.r2c(scale=SCALE)
    want = np.fft.rfftn(real.astype("f8")) * (SCALE / n)
    assert _spec_err(c.numpy(), want, dtype, n) <= 1
    c.value.mul_(1.0 / SCALE)
    back = c.c2r().numpy()
    assert _real_err(back, real.astype("f8"), dtype, n) <= 1


class _TwoRanks(object):
    """the communicator of rank 0 of two: enough for a ParticleMesh whose transform fails its checks before any
    exchange"""
    size, rank = 2, 0


def test_pow2_limit_checked_before_the_distributed_r2c(cuda, monkeypatch):
    """on P > 1 the x lines run last: an f8 mesh with 8192-point x lines must raise before the z and y passes launch"""
    from nbodykit_b200._lib import NbkError
    from nbodykit_b200.pmesh.pm import ParticleMesh, RealField
    monkeypatch.setenv("NBK_FFT_TRANSPOSE", "nccl")
    pm = ParticleMesh(BoxSize=1.0, Nmesh=[8192, 2, 4], dtype="f8", comm=_TwoRanks())
    f = RealField(pm)
    n0 = _lib().launch_count()
    with pytest.raises(NbkError, match="at most 4096"):
        f.r2c()
    assert _lib().launch_count() == n0
