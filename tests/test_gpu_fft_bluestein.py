"""
The Bluestein FFT (sides with a prime factor above 7) on the GPU: the line pass and the z pass against NumPy and, at
7-smooth lengths, against the mixed-radix passes; whole-mesh r2c / c2r through RealField / ComplexField; the slab route
of two virtual ranks on one GPU; and the algorithms above the field (FFTPower, FFTCorr, FFTRecon, ConvolvedFFTPower,
compute(Nmesh=), LogNormalCatalog) at such sizes against the CPU oracle.  Tolerances are those of test_gpu_fft_mixed.py
(f8 1e-13, f4 2e-6, times rms times log2 n).
"""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import pmesh_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = {"f8": 1e-13, "f4": 2e-6}
RTOL = 1e-5


def _vp(t):
    return ctypes.c_void_p(t.data_ptr())


def _code(dtype):
    return 4 if dtype == "f4" else 8


def _cdt(dtype):
    import torch
    return torch.complex64 if dtype == "f4" else torch.complex128


def _pm(N, L, dtype):
    from nbodykit_b200.pmesh.pm import ParticleMesh
    from nbodykit_b200.comm import SelfComm
    return ParticleMesh(BoxSize=L, Nmesh=N, dtype=dtype, comm=SelfComm())


def _err(got, want, dtype, n):
    """max error in units of the tolerance tol * rms(want) * log2(n)"""
    rms = np.sqrt((np.abs(want) ** 2).mean())
    return np.abs(got - want).max() / (TOL[dtype] * rms * max(np.log2(n), 2.0))


# primes, twice primes, 4094 = 2 23 89, and the 7-smooth 96 and 4096 (both paths valid there)
LINES = [11, 13, 17, 22, 26, 97, 127, 211, 509, 1009, 1021, 2039, 2053, 4093, 4094, 96, 4096]


@pytest.mark.parametrize("n", LINES)
@pytest.mark.parametrize("n_inner", [1, 9, 17])
@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_line_pass_vs_numpy(cuda, n, n_inner, dtype):
    """nbk_fft_lines_bluestein along the middle axis of [2][n][n_inner] (ragged column tiles at 9 and 17), in place and
    out of place, forward and inverse, with a scale"""
    import torch
    from nbodykit_b200 import _lib
    L = _lib.lib()
    rng = np.random.RandomState(n * 31 + n_inner)
    x = (rng.standard_normal((2, n, n_inner)) + 1j * rng.standard_normal((2, n, n_inner))).astype(
        np.complex64 if dtype == "f4" else np.complex128)
    fwd = np.fft.fft(x.astype(np.complex128), axis=1)
    inv = np.fft.ifft(x.astype(np.complex128), axis=1) * n
    smooth = n in (96, 4096)
    for inverse, want0 in ((0, fwd), (1, inv)):
        for inplace in (True, False):
            scale = 0.75
            src = torch.from_numpy(x.copy()).cuda()
            dst = src if inplace else torch.full_like(src, complex(np.nan, np.nan))
            _lib.check(L.nbk_fft_lines_bluestein(_vp(src), _vp(dst), _code(dtype), n, n_inner, n_inner, 2, n * n_inner, inverse,
                                                 scale, None), "nbk_fft_lines_bluestein")
            torch.cuda.synchronize()
            got = dst.cpu().numpy()
            e = _err(got, scale * want0, dtype, n)
            assert e <= 1.0, (inverse, inplace, e)
            if not inplace:
                np.testing.assert_array_equal(src.cpu().numpy(), x)        # the source is only read
            if smooth:
                ref = torch.from_numpy(x.copy()).cuda()
                _lib.check(L.nbk_fft_lines_mixed(_vp(ref), _vp(ref), _code(dtype), n, n_inner, n_inner, 2, n * n_inner, inverse,
                                                 scale, None), "nbk_fft_lines_mixed")
                torch.cuda.synchronize()
                assert _err(got, ref.cpu().numpy(), dtype, n) <= 1.0


ZS = [11, 13, 22, 26, 202, 1010, 1021, 4093, 8186]


@pytest.mark.parametrize("nz", ZS)
@pytest.mark.parametrize("rows", [1, 7])
@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_z_pass_vs_numpy(cuda, nz, rows, dtype):
    """nbk_fft_z_bluestein: rows of nz reals <-> nz/2+1 modes (odd row counts leave a half-filled row pair for odd nz)"""
    import torch
    from nbodykit_b200 import _lib
    L = _lib.lib()
    rng = np.random.RandomState(nz + rows)
    x = rng.standard_normal((rows, nz)).astype(dtype)
    nzc = nz // 2 + 1
    want = np.fft.rfft(x.astype("f8"), axis=1)
    real = torch.from_numpy(x).cuda()
    cplx = torch.empty((rows, nzc), dtype=_cdt(dtype), device="cuda")
    _lib.check(L.nbk_fft_z_bluestein(_vp(real), _vp(cplx), _code(dtype), rows, nz, 0, 0.5, None), "nbk_fft_z_bluestein")
    torch.cuda.synchronize()
    assert _err(cplx.cpu().numpy(), 0.5 * want, dtype, nz) <= 1.0
    np.testing.assert_array_equal(real.cpu().numpy(), x)
    # inverse: unnormalised, times scale
    spec = want.astype(np.complex64 if dtype == "f4" else np.complex128)
    c = torch.from_numpy(spec.copy()).cuda()
    back = torch.full((rows, nz), np.nan, dtype=real.dtype, device="cuda")
    _lib.check(L.nbk_fft_z_bluestein(_vp(c), _vp(back), _code(dtype), rows, nz, 1, 2.0, None), "nbk_fft_z_bluestein(inverse)")
    torch.cuda.synchronize()
    want_b = 2.0 * np.fft.irfft(spec.astype(np.complex128), n=nz, axis=1) * nz
    assert _err(back.cpu().numpy(), want_b, dtype, nz) <= 1.0
    np.testing.assert_array_equal(c.cpu().numpy(), spec)


SHAPES = [([11, 13, 17], "f8"), ([11, 13, 17], "f4"), ([22, 26, 34], "f8"), ([22, 26, 34], "f4"), ([44, 48, 37], "f8"),
          ([44, 48, 37], "f4"), ([97, 4, 6], "f8"), ([97, 4, 6], "f4"), ([6, 101, 10], "f8"), ([6, 101, 10], "f4"),
          ([176, 176, 176], "f4")]


@pytest.mark.parametrize("N,dtype", SHAPES)
def test_r2c_c2r_bluestein(cuda, N, dtype):
    """RealField.r2c == rfftn / N^3, ComplexField.c2r gives the input back, and both keep their input"""
    from nbodykit_b200.pmesh.pm import RealField
    rng = np.random.RandomState(5)
    real = rng.standard_normal(N).astype(dtype)
    pm = _pm(N, 1.0, dtype)
    assert any(pm.bluestein)
    f = RealField(pm)
    f[...] = real
    c = f.r2c()
    np.testing.assert_array_equal(f.numpy(), real)
    want = np.fft.rfftn(real.astype("f8")) / real.size
    got = c.numpy()
    assert got.shape == want.shape
    assert _err(got, want, dtype, real.size) <= 1.0
    back = c.c2r().numpy()
    assert np.abs(back - real).max() <= TOL[dtype] * 10 * np.log2(real.size)
    np.testing.assert_array_equal(c.numpy(), got)          # the complex input of c2r is preserved


def test_sides_beyond_the_line_limits_raise(cuda):
    """a side with a prime factor above 7 that is longer than the line limits raises with a message naming them"""
    from nbodykit_b200 import _lib
    from nbodykit_b200.pmesh.pm import RealField
    for N, want in (([4099, 4, 4], b"2 .. 4096"), ([4, 4, 8194], b"8192")):
        f = RealField(_pm(N, 1.0, 'f4'))
        f[...] = 1.0
        with pytest.raises(_lib.NbkError, match=want.decode()):
            f.r2c()


def test_complex_dtype_mesh_at_bluestein_size(cuda):
    """dtype='c16': r2c == fftn / N^3 over all modes"""
    from nbodykit_b200.pmesh.pm import RealField
    N = [22, 13, 26]
    pm = _pm(N, 1.0, 'c16')
    x = np.random.RandomState(3).normal(size=N)
    r = RealField(pm)
    r[...] = x
    c = r.r2c()
    assert not c.compressed and c.value.shape == tuple(N)
    np.testing.assert_allclose(c.value.cpu().numpy(), np.fft.fftn(x) / x.size, rtol=0, atol=1e-13)
    np.testing.assert_allclose(c.c2r().value.cpu().numpy(), x, rtol=0, atol=1e-12)


@pytest.mark.parametrize("shape", [(44, 22, 37), (26, 34, 22)])
@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_slab_route_two_virtual_ranks(cuda, dtype, shape):
    """the P > 1 route of RealField.r2c / ComplexField.c2r with two ranks simulated on one GPU, each pass the one
    ParticleMesh picks for its axis: z pass, y lines, nbk_transpose_pack; a block swap stands in for the all-to-all;
    nbk_transpose_unpack, x lines.  The result is rfftn; the inverse route gives the input back."""
    import torch
    from nbodykit_b200 import _lib
    L = _lib.lib()
    (Nx, Ny, Nz), P = shape, 2
    pm = _pm(list(shape), 1.0, dtype)
    assert any(pm.bluestein)
    zpass, ypass, xpass = pm._z_pass(), pm._line_pass(1), pm._line_pass(0)
    Nzc = Nz // 2 + 1
    x_n, y_n = Nx // P, Ny // P
    code, cdt = _code(dtype), _cdt(dtype)
    rng = np.random.RandomState(17)
    real = rng.standard_normal(shape).astype(dtype)
    want = np.fft.rfftn(real.astype("f8")) / real.size
    sends = []
    for r in range(P):
        slab = torch.from_numpy(real[r * x_n:(r + 1) * x_n].copy()).cuda()
        work = torch.empty((x_n, Ny, Nzc), dtype=cdt, device="cuda")
        send = torch.empty_like(work)
        _lib.check(zpass(_vp(slab), _vp(work), code, x_n * Ny, Nz, 0, 1.0, None))
        _lib.check(ypass(_vp(work), _vp(work), code, Ny, Nzc, Nzc, x_n, Ny * Nzc, 0, 1.0, None))
        _lib.check(L.nbk_transpose_pack(_vp(work), _vp(send), code, x_n, Ny, Nzc, P, None))
        sends.append(send.view(P, -1))
    outs = []
    for r in range(P):
        recv = torch.cat([sends[q][r] for q in range(P)])        # block r of every rank q, in rank order
        out = torch.empty((y_n, Nx, Nzc), dtype=cdt, device="cuda")
        _lib.check(L.nbk_transpose_unpack(_vp(recv), _vp(out), code, y_n, Nx, Nzc, P, None))
        _lib.check(xpass(_vp(out), _vp(out), code, Nx, Nzc, Nzc, y_n, Nx * Nzc, 0, 1.0 / real.size, None))
        torch.cuda.synchronize()
        ref = np.transpose(want[:, r * y_n:(r + 1) * y_n, :], (1, 0, 2))
        assert np.abs(out.cpu().numpy() - ref).max() <= TOL[dtype] * np.sqrt((np.abs(want) ** 2).mean()) * np.log2(real.size)
        outs.append(out)
    # inverse: x lines, pack_back, block swap, unpack_back, y lines, z pass
    backs = []
    for r in range(P):
        work = outs[r].clone()
        send = torch.empty_like(work)
        _lib.check(xpass(_vp(work), _vp(work), code, Nx, Nzc, Nzc, y_n, Nx * Nzc, 1, 1.0, None))
        _lib.check(L.nbk_transpose_pack_back(_vp(work), _vp(send), code, y_n, Nx, Nzc, P, None))
        backs.append(send.view(P, -1))
    for r in range(P):
        recv = torch.cat([backs[q][r] for q in range(P)])
        slab = torch.empty((x_n, Ny, Nzc), dtype=cdt, device="cuda")
        _lib.check(L.nbk_transpose_unpack_back(_vp(recv), _vp(slab), code, x_n, Ny, Nzc, P, None))
        _lib.check(ypass(_vp(slab), _vp(slab), code, Ny, Nzc, Nzc, x_n, Ny * Nzc, 1, 1.0, None))
        out = torch.empty((x_n, Ny, Nz), dtype=torch.float32 if dtype == "f4" else torch.float64, device="cuda")
        _lib.check(zpass(_vp(slab), _vp(out), code, x_n * Ny, Nz, 1, 1.0, None))
        torch.cuda.synchronize()
        assert np.abs(out.cpu().numpy() - real[r * x_n:(r + 1) * x_n]).max() <= TOL[dtype] * 10 * np.log2(real.size)


# ---- end to end, helpers as in test_gpu_fftpower.py
def _compare(r, o, mode):
    assert np.array_equal(r.power['modes'], np.squeeze(o['modes']))
    np.testing.assert_allclose(r.power['k'], np.squeeze(o['k']), rtol=RTOL, equal_nan=True)
    P, Po = r.power['power'], np.squeeze(o['power'])
    scale = np.nanmax(np.abs(Po))
    assert np.array_equal(np.isnan(P.real), np.isnan(Po.real))
    np.testing.assert_allclose(np.nan_to_num(P.real), np.nan_to_num(Po.real), rtol=RTOL, atol=RTOL * 1e-3 * scale)
    np.testing.assert_allclose(np.nan_to_num(P.imag), np.nan_to_num(Po.imag), rtol=RTOL, atol=RTOL * 1e-3 * scale)
    if mode == '2d':
        np.testing.assert_allclose(r.power['mu'], o['mu'], rtol=RTOL, atol=1e-7, equal_nan=True)


def test_fftpower_nmesh176_cic_tiled_paint(cuda):
    """Nmesh = 176 = 16 11 (multiple of 16: the tiled paint), CIC, f8, '1d'"""
    from nbodykit_b200.lab import UniformCatalog, FFTPower
    cat = UniformCatalog(nbar=3e-2, BoxSize=192., seed=42)      # 2e5 particles: above the tiled-paint thresholds
    assert cat.csize >= 2e5
    mesh = cat.to_mesh(Nmesh=176, resampler='cic', compensated=True, dtype='f8')
    r = FFTPower(mesh, mode='1d')
    pos, _ = po.uniform_catalog(3e-2, 192., 42)
    o = po.fftpower(pos, 176, 192., mode='1d', resampler='cic', compensated=True, dtype='f8')
    _compare(r, o, '1d')


def test_fftpower_44_52_37_tsc_interlaced_2d_poles(cuda):
    from nbodykit_b200.lab import UniformCatalog, FFTPower
    N = [44, 52, 37]
    cat = UniformCatalog(nbar=3e-4, BoxSize=512., seed=42)
    mesh = cat.to_mesh(Nmesh=N, resampler='tsc', interlaced=True, compensated=True, dtype='f4')
    r = FFTPower(mesh, mode='2d', Nmu=5, poles=[0, 2, 4], los=[0, 0, 1])
    pos, _ = po.uniform_catalog(3e-4, 512., 42)
    o = po.fftpower(pos, N, 512., mode='2d', resampler='tsc', interlaced=True, compensated=True, dtype='f4', Nmu=5,
                    poles=[0, 2, 4])
    assert np.array_equal(r.power['modes'], o['modes'])
    assert np.array_equal(r.poles['modes'], o['poles_modes'])
    np.testing.assert_allclose(r.power['k'], o['k'], rtol=RTOL, equal_nan=True)
    scale = np.nanmax(np.abs(o['poles_power'][0]))
    atol = 1e-5 * scale          # f4 meshes: wedges and ell > 0 multipoles measured against the monopole's amplitude
    np.testing.assert_allclose(np.nan_to_num(r.power['power'].real), np.nan_to_num(o['power'].real), rtol=RTOL, atol=atol)
    np.testing.assert_allclose(r.power['mu'], o['mu'], rtol=RTOL, atol=1e-7, equal_nan=True)
    for i, ell in enumerate([0, 2, 4]):
        np.testing.assert_allclose(np.nan_to_num(r.poles['power_%d' % ell].real), np.nan_to_num(o['poles_power'][i].real),
                                   rtol=RTOL, atol=atol)


def test_fftcorr_nmesh44(cuda):
    """FFTCorr at Nmesh = 44 against the numpy restatement of test_gpu_meshapi.py"""
    from nbodykit_b200.lab import UniformCatalog, FFTCorr
    from oracle import convpower_oracle as co
    N, L = 44, 256.
    cat = UniformCatalog(nbar=1e-3, BoxSize=L, seed=11)
    r = FFTCorr(cat.to_mesh(Nmesh=N, dtype='f8', resampler='cic', compensated=True), mode='2d', Nmu=4, poles=[0, 2])
    pos, _ = po.uniform_catalog(1e-3, L, 11)
    real, _ = po.paint_field(pos, N, L, 'cic', dtype='f8')
    c = po.compensate('CompensateCICShotnoise', po.k_coords(N, L, 'f4', kind='circular'), po.r2c(real))
    p3d = c * np.conj(c)
    p3d[0, 0, 0] = 0
    xi = po.c2r(p3d * L ** 3, N) / L ** 3
    dr = L / N
    redges = np.arange(0., 0.5 * L + dr / 2, dr)
    res, pres = po.project_to_basis(xi, co.x_coords(N, L, 'f4'), [redges, np.linspace(0, 1, 5)], poles=[0, 2],
                                    hermitian_symmetric=False)
    assert np.array_equal(r.corr['modes'], np.squeeze(res[3]))
    scale = np.nanmax(np.abs(res[2]))
    np.testing.assert_allclose(np.nan_to_num(r.corr['corr'].real), np.nan_to_num(np.squeeze(res[2]).real), rtol=1e-6,
                               atol=1e-7 * scale)
    np.testing.assert_allclose(np.nan_to_num(r.poles['corr_2'].real), np.nan_to_num(pres[1][1].real), rtol=1e-6,
                               atol=1e-7 * scale)


def test_fftrecon_nmesh44(cuda):
    from nbodykit_b200.lab import ArrayCatalog, FFTPower, FFTRecon
    from oracle import recon_oracle as ro
    N, L, R = 44, 400., 30.
    rng = np.random.RandomState(12)
    centres = rng.uniform(0, L, size=(300, 3))
    data = (centres[rng.randint(0, 300, size=20000)] + rng.standard_normal((20000, 3)) * 12.0) % L
    ran = rng.uniform(0, L, size=(60000, 3))
    dcat = ArrayCatalog({'Position': data}, BoxSize=L, Nmesh=N)
    rcat = ArrayCatalog({'Position': ran}, BoxSize=L, Nmesh=N)
    mesh = FFTRecon(data=dcat, ran=rcat, Nmesh=N, bias=1.5, f=0.4, los=[0, 0, 1], R=R, scheme='LRR')
    got = mesh.compute(mode='real').numpy()
    want, _, _ = ro.fftrecon(data, ran, N, L, bias=1.5, f=0.4, los=(0, 0, 1), R=R, scheme='LRR')
    assert np.abs(got - want).max() <= 1e-4 * np.abs(want).max()
    r = FFTPower(mesh, mode='1d')
    o = po.power_from_complex(po.r2c(want), None, N, L, mode='1d')
    assert np.array_equal(r.power['modes'], np.squeeze(o['modes']))
    np.testing.assert_allclose(r.power['power'].real, np.squeeze(o['power']).real, rtol=2e-4)


NBAR = 3e-4


def _fkp():
    from nbodykit_b200.lab import UniformCatalog, FKPCatalog
    d = UniformCatalog(nbar=NBAR, BoxSize=512., seed=42)
    r = UniformCatalog(nbar=10 * NBAR, BoxSize=512., seed=84)
    for c in (d, r):
        c['Position'] = c['Position'] + np.array((1000., -300., 700.))
        c['NZ'] = NBAR
    d['Weight'] = np.random.RandomState(5).uniform(0.8, 1.2, size=d.size)
    return FKPCatalog(d, r, P0=1e4), d, r


@pytest.mark.parametrize("dtype", ["c16", "f8"])
def test_convolved_power_nmesh44(cuda, dtype):
    from nbodykit_b200.lab import ConvolvedFFTPower
    from oracle import convpower_oracle as co
    fkp, d, r = _fkp()
    mesh = fkp.to_mesh(Nmesh=44, dtype=dtype)
    poles = [0, 1, 2] if dtype == "c16" else [0, 2, 4]
    res = ConvolvedFFTPower(mesh, poles=poles, dk=0.02)
    C, L = mesh.attrs['BoxCenter'], mesh.attrs['BoxSize']
    wfd = 1. / (1 + 1e4 * NBAR)
    args = (np.asarray(d['Position']), np.asarray(r['Position']),
            (np.asarray(d['Weight']), wfd * np.ones(d.size)), (np.ones(r.size), wfd * np.ones(r.size)),
            NBAR * np.ones(d.size), NBAR * np.ones(r.size), 44, L, C, poles)
    o = co.convpower_full(*args, dk=0.02) if dtype == "c16" else co.convpower(*args, dk=0.02)
    assert np.array_equal(res.poles['modes'], o['modes'])
    np.testing.assert_allclose(res.poles['k'], o['k'], rtol=1e-6, equal_nan=True)
    scale = np.nanmax(np.abs(o['power_0']))
    for ell in poles:
        got, want = res.poles['power_%d' % ell], o['power_%d' % ell]
        for part in ('real', 'imag'):
            np.testing.assert_allclose(np.nan_to_num(getattr(got, part)), np.nan_to_num(getattr(want, part)), rtol=1e-5,
                                       atol=2e-6 * scale)


def test_compute_at_nmesh44_resamples(cuda):
    """compute(Nmesh=44) of a 32^3 ArrayMesh reproduces a band-limited field"""
    from nbodykit_b200.lab import ArrayMesh
    N, L, M = 32, 64., 44
    x = np.arange(N) * (L / N)
    X, Y, Z = np.meshgrid(x, x, x, indexing='ij')

    def f(X, Y, Z):
        q = 2 * np.pi / L
        return 1.5 + np.cos(2 * q * X) * np.sin(3 * q * Y + 0.3) + 0.25 * np.cos(q * (X - 2 * Y + 4 * Z))
    mesh = ArrayMesh(f(X, Y, Z), BoxSize=L)
    xm = np.arange(M) * (L / M)
    Xm, Ym, Zm = np.meshgrid(xm, xm, xm, indexing='ij')
    got = mesh.compute(mode='real', Nmesh=M)
    assert got.value.shape == (M, M, M)
    np.testing.assert_allclose(got.numpy(), f(Xm, Ym, Zm), rtol=0, atol=1e-12)
    c = mesh.compute(mode='complex', Nmesh=M)
    assert c.value.shape == (M, M, M // 2 + 1)
    np.testing.assert_allclose(c.value[0, 0, 0].item().real, 1.5, rtol=1e-13)


def test_lognormal_catalog_nmesh44_reproducible(cuda):
    import torch
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.cosmology import NoWiggleEHPower
    from nbodykit_b200.source.catalog.lognormal import LogNormalCatalog
    kw = dict(Plin=NoWiggleEHPower(), nbar=2e-3, BoxSize=512., Nmesh=44, bias=2.0, seed=7, growth_rate=0.5, comm=SelfComm())
    cat = LogNormalCatalog(**kw)
    n = cat.csize
    assert abs(n / (2e-3 * 512. ** 3) - 1) < 0.1
    pos = cat['Position'].compute()
    assert float(pos.min()) >= 0.0 and float(pos.max()) < 512.
    again = LogNormalCatalog(**kw)
    assert again.csize == n and torch.equal(again['Position'].compute(), pos)


def test_reference_assertions_chi2_nmesh88(cuda):
    """algorithms/tests/test_fftpower.py:12-44 at Nmesh = 88 = 8 11: compensated CIC/TSC shot-noise spectra have
    reduced chi^2 < 1 over the bins the reference's 64^3 test covers (k below its Nyquist frequency, pi 64 / 512); the
    full-range value is pinned to the CPU oracle's, as in test_gpu_fft_mixed.py at 96."""
    from nbodykit_b200.lab import UniformCatalog, FFTPower
    pos, _ = po.uniform_catalog(3e-4, 512., 42)

    def chi2(Pk, modes, shotnoise):
        err = (2 * Pk ** 2 / modes) ** 0.5
        return ((Pk - shotnoise) / err) ** 2
    for resampler in ['cic', 'tsc']:
        source = UniformCatalog(nbar=3e-4, BoxSize=512., seed=42)
        mesh = source.to_mesh(resampler=resampler, Nmesh=88, compensated=True)
        r = FFTPower(mesh, mode='1d', kmin=0.02)
        c = chi2(r.power['power'].real, r.power['modes'], r.attrs['shotnoise'])
        sel = r.power['k'] < np.pi * 64 / 512.
        assert c[sel].mean() < 1.0, (resampler, c[sel].mean())       # "should be about 0.5-0.6"
        o = po.fftpower(pos, 88, 512., mode='1d', resampler=resampler, compensated=True, dtype='f4', kmin=0.02)
        co = chi2(np.squeeze(o['power']).real, np.squeeze(o['modes']), o['attrs']['shotnoise'])
        np.testing.assert_allclose(c.mean(), co.mean(), rtol=1e-5)


def test_two_gpu_fftpower_bluestein_matches_one_gpu():
    """launches tests/mgpu_check_bluestein.py under torchrun when the box has >= 2 GPUs"""
    import torch
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29521", os.path.join(ROOT, "tests", "mgpu_check_bluestein.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    sys.stdout.write(out.stdout[-3000:])
    sys.stderr.write(out.stderr[-3000:])
    assert out.returncode == 0
