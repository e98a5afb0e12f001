"""
The c2r contract on every FFT path: ComplexField.c2r(X) == scipy.fft.irfftn(X, s=N) * prod(N) for ANY half spectrum X
[Nx][Ny][Nz/2+1], complex everywhere, no symmetry assumed.  irfftn runs complex inverses along x and y, then a real
inverse along z that drops the imaginary parts of the kz = 0 entry and, for even Nz, of the kz = Nz/2 entry; FFTW's c2r
(behind pmesh, the reference's transform) follows the same rule.  Every reference here is float64 NumPy / SciPy or the
CPU oracle (oracle/pmesh_oracle.py, oracle/recon_oracle.py).

1. each inverse z pass alone -- power of two (nbk_fft_zy_backward on Ny = 1, so the y pass is the identity), mixed radix
   and Bluestein (nbk_fft_z_mixed / nbk_fft_z_bluestein, inverse = 1, scale != 1): rows whose only non-zero values are
   Im X[0] and Im X[Nz/2] give exactly zero, random complex rows give irfft;
2. ComplexField.c2r on one GPU, in every kernel regime of the three paths, and an exact known answer;
3. the distributed inverses: the peer and all-to-all routes of the power-of-two transform and the all-to-all route of the
   mixed-radix and Bluestein passes on virtual ranks of one process, and ComplexField.c2r on P = 2 and 3 gloo ranks;
4. pipelines that make spectra without the symmetry of a real field's: 1j k_d v filters, FFTRecon with R below the cell
   size, the Zel'dovich displacements of the mock maker, Fourier resampling to an even side.
"""
import numpy as np
import pytest
import scipy.fft
from gpu_helpers import code as _code, dev as _dev, host as _host, nbk as _lib, ptr as _p
from test_gpu_fft_bluestein import _err
from test_gpu_fft_mixed import _pm
from test_gpu_resample import _rule
from test_gpu_slab_fft import ROUTES, SLAB_CASES, TOL, _ids, _join_x, _rdt, _split_y
from test_gpu_slab_route import _spawn

from oracle import pmesh_oracle as po
from oracle import recon_oracle as ro

pytestmark = pytest.mark.gpu


def _cplx(dtype):
    return "c8" if dtype == "f4" else "c16"


def _spectrum(shape, dtype, seed):
    """unit-variance complex values in every entry: no Hermitian symmetry anywhere"""
    rng = np.random.RandomState(seed)
    return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(_cplx(dtype))


def _dc_nyquist(shape, nz, dtype):
    """zero except purely imaginary values at (0, 0, 0) and, for even Nz, (0, 0, Nz/2): the x and y inverses leave them
    purely imaginary on every (x, y) line, so the z pass must give exactly zero"""
    c = np.zeros(shape, dtype=_cplx(dtype))
    c[0, 0, 0] = 1.5j
    if nz % 2 == 0:
        c[0, 0, nz // 2] = -0.75j
    return c


def _irfftn(c, N):
    N = tuple(int(v) for v in N)
    return scipy.fft.irfftn(c.astype("c16"), s=N, axes=(0, 1, 2)) * float(np.prod(N))


def _real_err(got, want, dtype, n):
    """max error in units of the c2r tolerance of the FFT suites, TOL x 10 log2(n), scaled by rms(want)"""
    return np.abs(got - want).max() / (TOL[dtype] * 10 * np.log2(n) * np.sqrt((want ** 2).mean()))


def _n(N):
    return int(np.prod(N))


# ---------------------------------------------------------------------------------------------
# 1. the inverse z passes alone
# ---------------------------------------------------------------------------------------------
# (path, Nz): power-of-two rows from the shortest (4) to a long 8192; mixed-radix rows of 2 and 3 points, even and odd,
# 6000; Bluestein rows with odd and even Nz (2 x prime, 2 x 5 x 101, 2 x 4093)
Z_CASES = ([("pow2", nz) for nz in (4, 8, 64, 256, 512, 1024, 4096, 8192)]
           + [("mixed", nz) for nz in (2, 3, 6, 9, 12, 45, 100, 2187, 6000)]
           + [("bluestein", nz) for nz in (11, 13, 22, 26, 1010, 1021, 4093, 8186)])
Z_SCALE = {"pow2": 1.0, "mixed": 2.0, "bluestein": 0.75}      # the power-of-two pass takes no scale


def _z_inverse(path, c, nz, dtype):
    """the inverse z pass of `path` on rows c [rows][Nz/2+1] -> real rows [rows][Nz], unnormalised, times Z_SCALE"""
    import torch
    L = _lib()
    rows = c.shape[0]
    src = _dev(c)
    out = torch.full((rows, nz), float("nan"), dtype=_rdt(dtype), device="cuda")
    if path == "pow2":
        L.check(L.lib().nbk_fft_zy_backward(_p(src), _p(out), _code(dtype), rows, 1, nz, None), "fft_zy_backward")
    else:
        fn = L.lib().nbk_fft_z_mixed if path == "mixed" else L.lib().nbk_fft_z_bluestein
        L.check(fn(_p(src), _p(out), _code(dtype), rows, nz, 1, Z_SCALE[path], None), "fft_z(inverse)")
    return _host(out)


@pytest.mark.parametrize("path,nz", Z_CASES, ids=lambda v: str(v))
@pytest.mark.parametrize("rows", [1, 7])
@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_z_pass_drops_imaginary_dc_and_nyquist(cuda, path, nz, rows, dtype):
    """rows whose only non-zero values are Im X[0] and (even Nz) Im X[Nz/2] give zero, bit for bit (an odd row count
    leaves half a row pair at odd Nz)"""
    rng = np.random.RandomState(nz + rows)
    c = np.zeros((rows, nz // 2 + 1), dtype=_cplx(dtype))
    c[:, 0] = 1j * rng.uniform(0.5, 2.0, rows)
    if nz % 2 == 0:
        c[:, nz // 2] = -1j * rng.uniform(0.5, 2.0, rows)
    got = _z_inverse(path, c, nz, dtype)
    assert (got == 0).all(), "max |x| = %g" % np.abs(got).max()


@pytest.mark.parametrize("path,nz", Z_CASES, ids=lambda v: str(v))
@pytest.mark.parametrize("rows", [1, 7])
@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_z_pass_general_rows_equal_irfft(cuda, path, nz, rows, dtype):
    """random complex rows (complex X[0] and X[Nz/2] included) give scale irfft(X) Nz"""
    c = _spectrum((rows, nz // 2 + 1), dtype, 3 * nz + rows)
    want = Z_SCALE[path] * scipy.fft.irfft(c.astype("c16"), n=nz, axis=1) * nz
    got = _z_inverse(path, c, nz, dtype)
    assert _err(got, want, dtype, nz) <= 1.0


# ---------------------------------------------------------------------------------------------
# 2. ComplexField.c2r on one GPU
# ---------------------------------------------------------------------------------------------
MESH_SHAPES = [
    # power of two: Nz = 4, lines below 64 (shared-memory kernels), 64 / 128 (register I/O), 256 / 512 / 1024 (the TMA
    # line pass) on x and on y, long z rows, non-cubic throughout
    (8, 4, 4), (16, 32, 8), (64, 128, 4), (256, 4, 16), (4, 512, 8), (1024, 2, 4), (2, 4, 4096), (8, 16, 1024),
    # mixed radix: even and odd Nz, 6000-point rows, 1536-point y lines
    (12, 10, 6), (6, 10, 9), (45, 12, 15), (96, 48, 20), (4, 1536, 10), (2, 6, 6000),
    # Bluestein on every axis (odd and even Nz), on z alone (even and odd), on y alone
    (11, 13, 17), (22, 26, 34), (44, 48, 37), (8, 12, 22), (6, 10, 13), (6, 101, 10),
]


def _mesh_id(N):
    return "%dx%dx%d" % tuple(N)


def _c2r_one(N, c, dtype):
    from nbodykit_b200.pmesh.pm import ComplexField
    f = ComplexField(_pm(list(N), 1.0, dtype))
    f[...] = c
    got = f.c2r().numpy()
    np.testing.assert_array_equal(f.numpy(), c)          # c2r keeps its input
    return got


@pytest.mark.parametrize("N", MESH_SHAPES, ids=_mesh_id)
@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_mesh_c2r_general_spectrum(cuda, N, dtype):
    c = _spectrum((N[0], N[1], N[2] // 2 + 1), dtype, sum(N))
    got = _c2r_one(N, c, dtype)
    assert _real_err(got, _irfftn(c, N), dtype, _n(N)) <= 1.0


KNOWN_SHAPES = [(8, 8, 4), (16, 4, 8), (4, 2, 64), (12, 10, 6), (6, 10, 9), (8, 12, 22), (6, 10, 13), (22, 26, 34),
                (11, 13, 17)]


@pytest.mark.parametrize("N", KNOWN_SHAPES, ids=_mesh_id)
@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_mesh_c2r_drops_imaginary_dc_and_nyquist(cuda, N, dtype):
    """the spectrum of _dc_nyquist gives a field of zeros: bit for bit where the x and y passes are power-of-two or
    mixed-radix (their butterflies only add zeros and multiply by W^0 = 1 here), within rounding of |X| after Bluestein
    x / y passes, whose chirp products leave real parts of the order of the rounding error"""
    pm = _pm(list(N), 1.0, dtype)
    got = _c2r_one(N, _dc_nyquist((N[0], N[1], N[2] // 2 + 1), N[2], dtype), dtype)
    if pm.bluestein[0] or pm.bluestein[1]:
        assert np.abs(got).max() <= TOL[dtype] * 10 * np.log2(_n(N)) * 1.5
    else:
        assert (got == 0).all(), "max |x| = %g" % np.abs(got).max()


# ---------------------------------------------------------------------------------------------
# 3. distributed inverses
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", SLAB_CASES, ids=_ids)
@pytest.mark.parametrize("dtype", ["f8", "f4"])
@pytest.mark.parametrize("route", sorted(ROUTES))
def test_slab_routes_c2r_general_spectrum(cuda, case, dtype, route):
    """the peer and all-to-all inverses of the power-of-two transform on P virtual ranks: irfftn N^3 of a spectrum with
    no symmetry, and zeros, bit for bit, from the purely imaginary DC and Nyquist entries of rank 0's slab"""
    Nx, Ny, Nz, P = case
    N = (Nx, Ny, Nz)
    inv = ROUTES[route][1]
    c = _spectrum((Nx, Ny, Nz // 2 + 1), dtype, 11 + sum(case))
    got = _join_x(inv(_split_y(c, P), N, P, dtype))
    assert _real_err(got, _irfftn(c, N), dtype, _n(N)) <= 1.0
    got = _join_x(inv(_split_y(_dc_nyquist(c.shape, Nz, dtype), P), N, P, dtype))
    assert (got == 0).all(), "max |x| = %g" % np.abs(got).max()


def _inverse_passes(specs, N, P, dtype):
    """the all-to-all inverse of a mesh that is not all powers of two on P virtual ranks, each pass the one
    ParticleMesh picks for its axis (pm.py ComplexField._c2r_mixed): x lines, pack_back, block swap, unpack_back, y
    lines, z pass"""
    import torch
    L = _lib()
    Nx, Ny, Nz = N
    x_n, y_n, Nzc = Nx // P, Ny // P, Nz // 2 + 1
    pm = _pm(list(N), 1.0, dtype)
    code = _code(dtype)
    sends = []
    for r in range(P):
        work = specs[r].clone()
        L.check(pm._line_pass(0)(_p(work), _p(work), code, Nx, Nzc, Nzc, y_n, Nx * Nzc, 1, 1.0, None), "fft_lines(x)")
        send = torch.empty_like(work)
        L.check(L.lib().nbk_transpose_pack_back(_p(work), _p(send), code, y_n, Nx, Nzc, P, None), "pack_back")
        sends.append(send.view(P, -1))
    out = []
    for r in range(P):
        recv = torch.cat([sends[q][r] for q in range(P)])        # block r of every rank q, in rank order
        slab = torch.empty((x_n, Ny, Nzc), dtype=specs[r].dtype, device="cuda")
        L.check(L.lib().nbk_transpose_unpack_back(_p(recv), _p(slab), code, x_n, Ny, Nzc, P, None), "unpack_back")
        L.check(pm._line_pass(1)(_p(slab), _p(slab), code, Ny, Nzc, Nzc, x_n, Ny * Nzc, 1, 1.0, None), "fft_lines(y)")
        o = torch.empty((x_n, Ny, Nz), dtype=_rdt(dtype), device="cuda")
        L.check(pm._z_pass()(_p(slab), _p(o), code, x_n * Ny, Nz, 1, 1.0, None), "fft_z")
        out.append(o)
    return out


# (Nx, Ny, Nz, P): mixed radix with even and odd Nz at P = 2 and 3, Bluestein with odd and even Nz
SLAB_PASS_CASES = [(96, 48, 20, 2), (12, 30, 9, 3), (12, 30, 10, 3), (44, 22, 37, 2), (26, 34, 22, 2)]


@pytest.mark.parametrize("case", SLAB_PASS_CASES, ids=_ids)
@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_slab_passes_c2r_general_spectrum(cuda, case, dtype):
    Nx, Ny, Nz, P = case
    N = (Nx, Ny, Nz)
    c = _spectrum((Nx, Ny, Nz // 2 + 1), dtype, 5 + sum(case))
    got = _join_x(_inverse_passes(_split_y(c, P), N, P, dtype))
    assert _real_err(got, _irfftn(c, N), dtype, _n(N)) <= 1.0
    got = _join_x(_inverse_passes(_split_y(_dc_nyquist(c.shape, Nz, dtype), P), N, P, dtype))
    if any(_pm(list(N), 1.0, dtype).bluestein[:2]):         # as in test_mesh_c2r_drops_imaginary_dc_and_nyquist
        assert np.abs(got).max() <= TOL[dtype] * 10 * np.log2(_n(N)) * 1.5
    else:
        assert (got == 0).all(), "max |x| = %g" % np.abs(got).max()


def _c2r_ranks(comm, N, specs):
    """ComplexField.c2r of each spectrum on this rank's transposed y slab; returns this rank's x slabs"""
    import torch
    from nbodykit_b200.pmesh.pm import ComplexField, ParticleMesh
    out = {}
    for key, c in specs.items():
        pm = ParticleMesh(BoxSize=1.0, Nmesh=list(N), dtype="f4" if c.dtype == np.complex64 else "f8", comm=comm)
        f = ComplexField(pm)
        mine = np.ascontiguousarray(c[:, pm.y_start:pm.y_start + pm.y_n].transpose(1, 0, 2))
        f.value.copy_(torch.from_numpy(mine).cuda())
        out[key] = f.c2r().numpy()
    return out


@pytest.mark.parametrize("N,P", [((32, 16, 8), 2), ((12, 30, 10), 3), ((12, 30, 9), 3), ((44, 22, 26), 2)],
                         ids=lambda v: str(v))
def test_gloo_ranks_c2r_general_spectrum(cuda, N, P):
    """ComplexField.c2r on P processes sharing device 0 (all-to-all transpose): power of two, mixed radix with even and
    odd Nz, Bluestein"""
    specs = {}
    for dtype in ("f8", "f4"):
        specs["rand-" + dtype] = _spectrum((N[0], N[1], N[2] // 2 + 1), dtype, 17 + sum(N))
        specs["dc-" + dtype] = _dc_nyquist((N[0], N[1], N[2] // 2 + 1), N[2], dtype)
    parts = _spawn(_c2r_ranks, P, N, specs)
    bluestein_xy = any(_pm(list(N), 1.0, "f8").bluestein[:2])
    for dtype in ("f8", "f4"):
        got = np.concatenate([p["rand-" + dtype] for p in parts])
        assert _real_err(got, _irfftn(specs["rand-" + dtype], N), dtype, _n(N)) <= 1.0, dtype
        got = np.concatenate([p["dc-" + dtype] for p in parts])
        if bluestein_xy:
            assert np.abs(got).max() <= TOL[dtype] * 10 * np.log2(_n(N)) * 1.5, dtype
        else:
            assert (got == 0).all(), "%s: max |x| = %g" % (dtype, np.abs(got).max())


# ---------------------------------------------------------------------------------------------
# 4. pipelines against the CPU oracle, Nyquist modes present
# ---------------------------------------------------------------------------------------------
# (Nmesh, BoxSize): power of two, mixed radix with even and odd Nz, Bluestein with even and odd Nz; Nx and Ny even for
# two ranks
DERIV_SHAPES = [((16, 32, 8), (100., 120., 80.)), ((12, 10, 18), (60., 50., 90.)), ((12, 10, 15), (60., 50., 75.)),
                ((22, 26, 34), (110., 130., 170.)), ((22, 26, 17), (110., 130., 85.))]
DERIV_AXES = (0, 2)


def _field(N, seed):
    """a white-noise field: every mode up to the Nyquist planes is populated"""
    return np.random.RandomState(seed).standard_normal(N)


def _deriv_oracle(a, N, L, d):
    k = po.k_coords(N, L)                          # the f4 wavenumbers ComplexField.apply hands a callback
    return po.c2r(1j * k[d] * po.r2c(a), N)


def _deriv_ranks(comm, a, L):
    """this rank's x slab of each derivative filter, f8 and f4 meshes"""
    from nbodykit_b200.lab import ArrayMesh
    out = {}
    for dtype in ("f8", "f4"):
        mesh = ArrayMesh(a.astype(dtype), BoxSize=L, comm=comm)
        for d in DERIV_AXES:
            out[dtype, d] = mesh.apply(lambda k, v, d=d: 1j * k[d] * v).compute(mode='real').numpy()
    return out


@pytest.mark.parametrize("N,L", DERIV_SHAPES, ids=lambda v: "x".join("%g" % x for x in v))
@pytest.mark.parametrize("P", [1, 2])
def test_derivative_filter_vs_oracle(cuda, N, L, P):
    """ArrayMesh(...).apply(lambda k, v: 1j k[d] v).compute(mode='real'), d = 0 and 2: at the Nyquist planes of an even
    side 1j k v is anti-Hermitian, and the c2r must drop what irfftn drops"""
    from nbodykit_b200.comm import SelfComm
    a = _field(N, sum(N))
    parts = [_deriv_ranks(SelfComm(), a, L)] if P == 1 else _spawn(_deriv_ranks, P, a, L)
    for dtype in ("f8", "f4"):
        for d in DERIV_AXES:
            got = np.concatenate([p[dtype, d] for p in parts])
            assert _real_err(got, _deriv_oracle(a, N, L, d), dtype, _n(N)) <= 1.0, (dtype, d)


@pytest.mark.parametrize("N", [32, 30, 27])
def test_fftrecon_small_smoothing_vs_oracle(cuda, N):
    """FFTRecon with R at half the cell size (the Nyquist modes keep 0.3 of their amplitude): the displacements of data
    and randoms, and the reconstructed mesh, against oracle/recon_oracle.py"""
    from nbodykit_b200.lab import ArrayCatalog, FFTRecon
    L = 400.
    R = 0.5 * L / N
    rng = np.random.RandomState(N)
    centres = rng.uniform(0, L, size=(300, 3))
    data = (centres[rng.randint(0, 300, size=20000)] + rng.standard_normal((20000, 3)) * 12.0) % L
    ran = rng.uniform(0, L, size=(60000, 3))
    dcat = ArrayCatalog({'Position': data}, BoxSize=L, Nmesh=N)
    rcat = ArrayCatalog({'Position': ran}, BoxSize=L, Nmesh=N)
    with pytest.warns(UserWarning, match="smoothing radius"):
        mesh = FFTRecon(data=dcat, ran=rcat, Nmesh=N, bias=1.5, f=0.4, los=[0, 0, 1], R=R, scheme='LRR')
    want, s_d, s_r = ro.fftrecon(data, ran, N, L, bias=1.5, f=0.4, los=(0, 0, 1), R=R, scheme='LRR')
    got_d, got_r = [s.cpu().numpy() for s in mesh._compute_s()]
    # f4 displacements read out at f4 positions: a few f4 roundings of max |s|
    for got, ref, name in ((got_d, s_d, "data"), (got_r, s_r, "randoms")):
        assert np.abs(got - ref).max() <= 1e-5 * np.abs(ref).max(), name
    got = mesh.compute(mode='real').numpy()
    assert np.abs(got - want).max() <= 1e-4 * np.abs(want).max()       # the bound of test_gpu_recon.py


@pytest.mark.parametrize("N", [32, 30, 27])
def test_mock_displacements_equal_irfftn(cuda, N):
    """gaussian_complex_fields(compute_displacement=True): the three psi spectra are anti-Hermitian on the Nyquist
    planes of an even side; their c2r must equal irfftn of the same spectra, and poisson_sample_to_points must carry
    those fields' value at each point's cell (nearest grid point) in its displacement column"""
    import torch
    from nbodykit_b200 import mockmaker
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.cosmology import NoWiggleEHPower
    from nbodykit_b200.pmesh.pm import ParticleMesh, RealField
    L = 200.
    pm = ParticleMesh(BoxSize=L, Nmesh=[N] * 3, dtype='f4', comm=SelfComm())     # LogNormalCatalog's generator mesh
    delta_k, disp_k = mockmaker.gaussian_complex_fields(pm, NoWiggleEHPower(), 7, compute_displacement=True)
    n = N ** 3
    fields, want = [], []
    for d in range(3):
        spec = disp_k[d].numpy()
        fields.append(disp_k[d].c2r())
        want.append(_irfftn(spec, [N] * 3))
        assert _real_err(fields[d].numpy(), want[d], "f4", n) <= 1.0, d
    delta = delta_k.c2r()
    # the cell of every point: the same draw with a "displacement" that holds the flat cell index (exact in f4)
    index = RealField(pm)
    index.value.copy_(torch.arange(n, dtype=torch.float32, device="cuda").view(N, N, N))
    nbar, seed = 1.0 / (L / N) ** 3, 99
    _, cells = mockmaker.poisson_sample_to_points(delta.copy(), [index] * 3, pm, nbar, bias=1.0, seed=seed)
    _, dsp = mockmaker.poisson_sample_to_points(delta.copy(), fields, pm, nbar, bias=1.0, seed=seed)
    cells = cells[:, 0].cpu().numpy().astype("i8")
    dsp = dsp.cpu().numpy()
    assert len(cells) > n // 2
    for d in range(3):
        np.testing.assert_array_equal(dsp[:, d], fields[d].numpy().reshape(-1)[cells])
        ref = want[d].reshape(-1)[cells]
        assert _real_err(dsp[:, d].astype("f8"), ref, "f4", n) <= 1.0, d


# (source side, destination side): down to an even side (the destination Nyquist planes take source modes that have no
# partner), up from an even side (its Nyquist row lands on the negative label only)
RESAMPLE_PAIRS = [(45, 32), (33, 20), ((30, 33, 17), (24, 22, 16)), (32, 48)]


@pytest.mark.parametrize("Ns,Nd", RESAMPLE_PAIRS, ids=lambda v: str(v))
@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_resample_to_even_side_vs_oracle(cuda, Ns, Nd, dtype):
    """compute(mode='real', Nmesh=Nd) and preview(Nmesh=Nd) of a white-noise field: the c2r of the resampled spectrum
    (the copy rule of test_gpu_resample.py) equals irfftn of it"""
    from nbodykit_b200.lab import ArrayMesh
    Ns = [int(v) for v in np.ones(3, 'i8') * Ns]
    Nd = [int(v) for v in np.ones(3, 'i8') * Nd]
    a = _field(Ns, 23).astype(dtype)
    mesh = ArrayMesh(a, BoxSize=64.)
    want = po.c2r(_rule(po.r2c(a.astype("f8")), Ns, Nd), Nd)
    got = mesh.compute(mode='real', Nmesh=Nd).numpy()
    assert got.shape == tuple(Nd)
    assert _real_err(got, want, dtype, _n(Nd)) <= 1.0
    got = mesh.preview(Nmesh=Nd, axes=(2, 0))
    ref = want.sum(axis=1).T
    assert _real_err(got, ref, dtype, _n(Nd)) <= 1.0
