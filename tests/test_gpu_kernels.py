"""
Parity of each CUDA kernel (through the C ABI, via the pmesh shim) against the CPU oracle.
Bit-exact for indices and mode counts; float tolerances are written at each assert.
"""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import pmesh_oracle as po

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _pm(N, L, dtype):
    from nbodykit_b200.pmesh.pm import ParticleMesh
    from nbodykit_b200.comm import SelfComm
    return ParticleMesh(BoxSize=L, Nmesh=N, dtype=dtype, comm=SelfComm())


def _particles(n, L, dtype, seed=7, outside=True):
    rng = np.random.RandomState(seed)
    pos = rng.uniform(0, 1, size=(n, 3)) * np.asarray(L)
    if outside:  # a few particles outside the box and exactly on nodes / the upper edge: wrap semantics
        pos[:5] += np.asarray(L)
        pos[5:10] -= np.asarray(L) * 2
        pos[10] = 0.0
        pos[11] = np.asarray(L) * (1 - 1e-12)
        pos[12] = np.asarray(L) / 2
    return pos.astype(dtype)


@pytest.mark.parametrize("resampler", ["nnb", "cic", "tsc", "pcs"])
@pytest.mark.parametrize("pos_dtype", ["f4", "f8"])
@pytest.mark.parametrize("shift", [0.0, 0.5])
def test_cell_index_bit_exact(cuda, resampler, pos_dtype, shift):
    N, L = [32, 16, 64], [100., 50., 731.]
    pos = _particles(20000, L, pos_dtype)
    pm = _pm(N, L, "f8")
    got = pm.cell_index(pos, resampler, shift).cpu().numpy()
    want = po.cell_index(pos, N, L, resampler, shift)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("resampler", ["nnb", "cic", "tsc", "pcs"])
@pytest.mark.parametrize("mesh_dtype,pos_dtype,tol", [("f8", "f8", 1e-12), ("f8", "f4", 1e-12), ("f4", "f4", 2e-5)])
@pytest.mark.parametrize("weighted", [False, True])
def test_paint_vs_oracle(cuda, resampler, mesh_dtype, pos_dtype, tol, weighted):
    N, L = [16, 32, 8], [64., 128., 10.]
    pos = _particles(30000, L, pos_dtype)
    mass = np.random.RandomState(3).uniform(0.5, 1.5, size=len(pos)) if weighted else None
    pm = _pm(N, L, mesh_dtype)
    got = pm.paint(pos, mass=mass if weighted else 1.0, resampler=resampler).numpy()
    want = po.paint(pos, mass, N, L, resampler, dtype="f8")
    # mass is conserved and every cell agrees: |diff| <= tol * max cell (f4: order-dependent adds)
    assert got.dtype == np.dtype(mesh_dtype)
    np.testing.assert_allclose(got, want, rtol=0, atol=tol * want.max())
    np.testing.assert_allclose(got.sum(dtype="f8"), (mass.sum() if weighted else len(pos)), rtol=1e-6)


def test_paint_hold_shift_and_scalar_mass(cuda):
    N, L = 16, 32.
    pos = _particles(5000, [L] * 3, "f8")
    pm = _pm(N, L, "f8")
    from nbodykit_b200.pmesh.pm import RealField
    out = RealField(pm)
    out[...] = 1.0
    pm.paint(pos, mass=2.5, resampler="tsc", transform=pm.affine.shift(0.5), hold=True, out=out)
    want = 1.0 + 2.5 * po.paint(pos, None, N, L, "tsc", shift=0.5)
    np.testing.assert_allclose(out.numpy(), want, rtol=0, atol=1e-12 * want.max())


def test_paint_slab_drops_ghost_planes(cuda):
    """x_start/x_n: stencil points outside the slab are dropped (pmesh ghost semantics)"""
    import ctypes
    import torch
    from nbodykit_b200 import _lib
    N, L = [16, 8, 8], [16., 8., 8.]
    pos = _particles(4000, L, "f8")
    full = po.paint(pos, None, N, L, "tsc")
    p = torch.from_numpy(pos).cuda()
    for x0, xn in [(0, 4), (4, 4), (12, 4), (5, 11)]:
        mesh = torch.zeros((xn, 8, 8), dtype=torch.float64, device="cuda")
        _lib.check(_lib.lib().nbk_paint(ctypes.c_void_p(p.data_ptr()), 8, len(pos), None, 8, 3, 0.0, _lib.darr(L),
                                        _lib.iarr(N), x0, xn, ctypes.c_void_p(mesh.data_ptr()), 8, None))
        torch.cuda.synchronize()
        np.testing.assert_allclose(mesh.cpu().numpy(), full[x0:x0 + xn], rtol=0, atol=1e-12 * full.max())


def test_paint_empty(cuda):
    pm = _pm(8, 1.0, "f4")
    out = pm.paint(np.empty((0, 3), dtype="f4"), resampler="cic")
    assert float(out.numpy().sum()) == 0.0


def test_paint_interlaced_pair(cuda):
    from nbodykit_b200.pmesh.pm import RealField
    N, L = 16, 100.
    pos = _particles(8000, [L] * 3, "f4")
    pm = _pm(N, L, "f4")
    r1, r2 = RealField(pm), RealField(pm)
    r1[...] = 0; r2[...] = 0
    pm.paint_interlaced(pos, None, "cic", r1, r2)
    w1 = po.paint(pos, None, N, L, "cic", 0.0)
    w2 = po.paint(pos, None, N, L, "cic", 0.5)
    np.testing.assert_allclose(r1.numpy(), w1, rtol=0, atol=2e-5 * w1.max())
    np.testing.assert_allclose(r2.numpy(), w2, rtol=0, atol=2e-5 * w2.max())


@pytest.mark.parametrize("N", [[8, 8, 8], [16, 32, 64], [64, 16, 4], [128, 128, 128], [2, 4, 8], [256, 64, 32], [512, 128, 16],
                               [1024, 8, 16], [2048, 4, 8],
                               # y / x lines of 256, 512, 1024: the TMA-pipelined line pass (ragged last column tile included)
                               [4, 256, 16], [2, 512, 8], [2, 1024, 8], [256, 256, 16], [512, 4, 16]])
@pytest.mark.parametrize("dtype,tol", [("f8", 1e-13), ("f4", 2e-6)])
def test_r2c_c2r(cuda, N, dtype, tol):
    from nbodykit_b200.pmesh.pm import RealField
    rng = np.random.RandomState(5)
    real = rng.standard_normal(N).astype(dtype)
    pm = _pm(N, 1.0, dtype)
    f = RealField(pm)
    f[...] = real
    c = f.r2c()
    want = np.fft.rfftn(real.astype("f8")) / real.size
    got = c.numpy()
    assert got.shape == want.shape
    # tolerance relative to the rms amplitude of the spectrum
    assert np.abs(got - want).max() <= tol * np.sqrt((np.abs(want) ** 2).mean()) * np.log2(real.size)
    back = c.c2r().numpy()
    assert np.abs(back - real).max() <= tol * 10 * np.log2(real.size)
    # the complex input of c2r is preserved
    np.testing.assert_array_equal(c.numpy(), got)


@pytest.mark.parametrize("N", [[8, 8, 256], [4, 8, 512], [4, 4, 1024], [2, 4, 2048], [4, 4, 4096]])
@pytest.mark.parametrize("dtype,tol", [("f8", 1e-13), ("f4", 2e-6)])
def test_r2c_long_rows(cuda, N, dtype, tol):
    """long z rows: packed lengths 128 .. 2048 cover every last-stage radix (8 / 4 / 2) of the register-I/O z pass"""
    from nbodykit_b200.pmesh.pm import RealField
    rng = np.random.RandomState(1)
    real = rng.standard_normal(N).astype(dtype)
    pm = _pm(N, 1.0, dtype)
    f = RealField(pm)
    f[...] = real
    got = f.r2c().numpy()
    want = np.fft.rfftn(real.astype("f8")) / real.size
    assert np.abs(got - want).max() <= tol * np.sqrt((np.abs(want) ** 2).mean()) * np.log2(real.size)


@pytest.mark.parametrize("name", sorted(["CompensateCIC", "CompensateTSC", "CompensatePCS", "CompensateCICShotnoise",
                                         "CompensateTSCShotnoise", "CompensatePCSShotnoise"]))
@pytest.mark.parametrize("dtype,tol", [("f8", 2e-6), ("f4", 3e-6)])
def test_compensate(cuda, name, dtype, tol):
    """oracle forms the factors in float32 (reference dtype flow); the kernel in f8 -> 1e-7-level agreement"""
    from nbodykit_b200.pmesh.pm import ComplexField
    N, L = [16, 8, 32], [10., 20., 30.]
    rng = np.random.RandomState(2)
    shape = (N[0], N[1], N[2] // 2 + 1)
    c = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype("c8" if dtype == "f4" else "c16")
    pm = _pm(N, L, dtype)
    f = ComplexField(pm)
    f[...] = c
    f.compensate(name)
    want = po.compensate(name, po.k_coords(N, L, "f4", kind="circular"), c)
    np.testing.assert_allclose(f.numpy(), want, rtol=tol, atol=0)
    # and against exact f8 factors: tight
    want8 = po.compensate(name, po.k_coords(N, L, "f8", kind="circular"), c.astype("c16"))
    np.testing.assert_allclose(f.numpy(), want8, rtol=1e-13 if dtype == "f8" else 2e-7, atol=0)


@pytest.mark.parametrize("dtype,tol", [("f8", 1e-13), ("f4", 3e-7)])
def test_interlace_combine(cuda, dtype, tol):
    from nbodykit_b200.pmesh.pm import ComplexField
    N, L = [8, 16, 32], [10., 20., 30.]
    rng = np.random.RandomState(4)
    shape = (N[0], N[1], N[2] // 2 + 1)
    cd = "c8" if dtype == "f4" else "c16"
    c1 = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(cd)
    c2 = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(cd)
    pm = _pm(N, L, dtype)
    f1, f2 = ComplexField(pm), ComplexField(pm)
    f1[...] = c1; f2[...] = c2
    f1.interlace_combine(f2)
    want = po.interlace_combine(c1.astype("c16"), c2.astype("c16"), N, L, "f8")
    assert np.abs(f1.numpy() - want).max() <= tol * 4


def _bin(pm, c, edges, los, poles, coord="f4", is_p3d=True, c2=None, volume=1.0):
    from nbodykit_b200.algorithms.fftpower import project_to_basis_device
    from nbodykit_b200.pmesh.pm import ComplexField
    f = ComplexField(pm)
    f[...] = c
    g = None
    if c2 is not None:
        g = ComplexField(pm)
        g[...] = c2
    return project_to_basis_device(f, edges, los=los, poles=poles, coord_dtype=coord, is_p3d=is_p3d, second=g,
                                   volume=volume)


@pytest.mark.parametrize("N,L", [([16, 16, 16], 64.), ([8, 16, 32], [10., 20., 30.]), ([32, 32, 32], 1024.)])
@pytest.mark.parametrize("dtype", ["f8", "f4"])
@pytest.mark.parametrize("Nmu,poles,los", [(1, [], [0, 0, 1]), (5, [0, 2, 4], [0, 0, 1]), (4, [1, 2], [0, 1, 0]),
                                           (3, [2], [0.6, 0, 0.8])])
@pytest.mark.parametrize("coord", ["f4", "f8"])
def test_power_bin_vs_oracle(cuda, N, L, dtype, Nmu, poles, los, coord):
    rng = np.random.RandomState(11)
    shape = (N[0], N[1], N[2] // 2 + 1)
    c = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype("c8" if dtype == "f4" else "c16")
    Lv = np.ones(3) * L
    dk = 2 * np.pi / Lv.min()
    kedges = np.arange(0., np.pi * min(N) / Lv.max() + dk / 2, dk)
    muedges = np.linspace(-1, 1, Nmu + 1)
    pm = _pm(N, L, dtype)
    res, pres = _bin(pm, c, [kedges, muedges], los, poles, coord)
    ores, opres = po.project_to_basis(c, po.k_coords(N, L, coord), [kedges, muedges], los=los, poles=poles)
    # mode counts: bit-exact
    assert np.array_equal(res[3], ores[3])
    tol = 1e-12 if dtype == "f8" else 2e-6
    for a, b in zip(res[:3], ores[:3]):
        assert np.array_equal(np.isnan(a), np.isnan(b))
        np.testing.assert_allclose(np.nan_to_num(a), np.nan_to_num(b), rtol=tol, atol=tol * np.nanmax(np.abs(b)))
    if poles:
        assert np.array_equal(pres[2], opres[2])
        np.testing.assert_allclose(np.nan_to_num(pres[0]), np.nan_to_num(opres[0]), rtol=tol)
        np.testing.assert_allclose(np.nan_to_num(pres[1]), np.nan_to_num(opres[1]), rtol=tol,
                                   atol=tol * np.nanmax(np.abs(opres[1])))


def test_power_bin_cross_and_zero_mode(cuda):
    """c1*conj(c2)*V with the k=0 mode cleared (fftpower.py:115-128) fused into the binning pass"""
    N, L = [16, 16, 16], 100.
    rng = np.random.RandomState(12)
    shape = (16, 16, 9)
    c1 = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape))
    c2 = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape))
    V = L ** 3
    p3d = c1 * np.conj(c2)
    p3d[0, 0, 0] = 0
    p3d *= V
    dk = 2 * np.pi / L
    kedges = np.arange(0., np.pi * 16 / L + dk / 2, dk)
    muedges = np.linspace(-1, 1, 6)
    pm = _pm(N, L, "f8")
    res, pres = _bin(pm, c1, [kedges, muedges], [0, 0, 1], [0, 2], "f4", is_p3d=False, c2=c2, volume=V)
    ores, opres = po.project_to_basis(p3d, po.k_coords(N, L, "f4"), [kedges, muedges], poles=[0, 2])
    assert np.array_equal(res[3], ores[3])
    np.testing.assert_allclose(np.nan_to_num(res[2]), np.nan_to_num(ores[2]), rtol=1e-12, atol=1e-12 * V)
    np.testing.assert_allclose(np.nan_to_num(pres[1]), np.nan_to_num(opres[1]), rtol=1e-12, atol=1e-12 * V)


def test_shell_counts_match_reference_fixture(cuda):
    """known-answer: k-marginal mode counts of nbodykit/tests/data/dataset_2d.json (128^3, L=512, dk=k_f)"""
    gold = json.load(open(os.path.join(GOLD, "dataset_2d_modes.json")))
    N, L = gold["Nmesh"], gold["BoxSize"]
    dk = 2 * np.pi / L
    kedges = np.arange(0., np.pi * N / L + dk / 2, dk)
    pm = _pm(N, L, "f4")
    c = np.ones((N, N, N // 2 + 1), dtype="c8")
    res, _ = _bin(pm, c, [kedges, np.linspace(-1, 1, 2)], [0, 0, 1], [], "f4")
    assert res[3][:, 0].tolist() == gold["modes_k"]
    # and through 5 mu bins the k-marginal is unchanged
    res5, _ = _bin(pm, c, [kedges, np.linspace(-1, 1, 6)], [0, 0, 1], [], "f4")
    assert res5[3].sum(axis=1).tolist() == gold["modes_k"]


def test_elementwise_and_sums(cuda):
    from nbodykit_b200.pmesh.pm import RealField
    pm = _pm([8, 4, 6], 1.0, "f4")   # 192 elements: exercises vector body; odd sizes below the tail
    f = RealField(pm)
    f[...] = 2.0
    f *= 1.5
    g = f.copy()
    g /= 3.0
    f += g
    assert np.allclose(f.numpy(), 4.0)
    assert abs(f.csum() - 4.0 * 192) < 1e-9
    assert abs(f.cmean() - 4.0) < 1e-12


# ---------------------------------------------------------------------------------------------
# tile-sorted shared-memory paint path (nbk_paint_tiled)
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("resampler", ["nnb", "cic", "tsc", "pcs"])
@pytest.mark.parametrize("mesh_dtype,pos_dtype", [("f8", "f4"), ("f4", "f4"), ("f8", "f8")])
@pytest.mark.parametrize("weighted", [False, True])
def test_paint_tiled_vs_oracle(cuda, resampler, mesh_dtype, pos_dtype, weighted):
    N, L = [32, 48, 64], [64., 100., 10.]
    pos = _particles(200000, L, pos_dtype)
    mass = None
    if weighted:   # includes negative and widely different masses
        mass = np.random.RandomState(3).uniform(-2.0, 3.0, size=len(pos))
    pm = _pm(N, L, mesh_dtype)
    got = pm.paint(pos, mass=mass if weighted else 1.0, resampler=resampler, method='tiled').numpy()
    want = po.paint(pos, mass, N, L, resampler, dtype="f8")
    amax = np.abs(want).max()
    # fixed point: 2^-31 of max|mass| per deposit; f4 meshes add the final cast
    tol = 1e-7 if mesh_dtype == "f8" else 3e-6
    np.testing.assert_allclose(got, want, rtol=0, atol=tol * amax)
    # agrees with the direct (REDG) path as well
    direct = pm.paint(pos, mass=mass if weighted else 1.0, resampler=resampler, method='direct').numpy()
    np.testing.assert_allclose(got, direct, rtol=0, atol=max(tol, 2e-5 if mesh_dtype == "f4" else 0) * amax)


@pytest.mark.parametrize("resampler,pos_dtype,weighted", [("cic", "f4", False), ("cic", "f8", True), ("tsc", "f4", True),
                                                          ("pcs", "f4", False), ("nnb", "f8", False)])
@pytest.mark.parametrize("knobs", [{}, {"NBK_PAINT_WSTAGE": "0"}, {"NBK_PAINT_DEFER_CAP": "700"}, {"NBK_PAINT_W": "16"}])
def test_paint_tiled_coherent_plan_variants(cuda, monkeypatch, resampler, pos_dtype, weighted, knobs):
    """the coherent bucketing plan (windowed histogram, per-warp record transposition) and the write-back variants of the
    tile pass (deferred halo list, its overflow -> wait fallback): cell-sorted input, and the same plan forced
    onto unsorted input; NBK_PAINT_W=16 shrinks the tile window below the 48 tiles of this mesh, so most particles take the
    out-of-window (global atomic) route; all must reproduce the oracle"""
    N, L = [64, 48, 64], [128., 96., 128.]                # power-of-two N/L on x and z, not on y: both record paths
    pos = _particles(250000, L, pos_dtype)
    mass = np.random.RandomState(11).uniform(-1.0, 2.0, size=len(pos)) if weighted else None
    g = np.floor(pos.astype("f8") * (np.array(N) / np.array(L))).astype("i8")
    order = np.lexsort((g[:, 2], g[:, 1], g[:, 0]))        # generator-like cell order
    pm = _pm(N, L, "f8")
    want = po.paint(pos, mass, N, L, resampler, dtype="f8")
    amax = np.abs(want).max()
    for k, v in knobs.items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("NBK_PAINT_BUCKET", "coherent")
    for idx in (order, np.arange(len(pos))):
        got = pm.paint(pos[idx], mass=mass[idx] if weighted else 1.0, resampler=resampler, method='tiled').numpy()
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-7 * amax)


def test_paint_tiled_is_order_independent(cuda):
    """fixed-point accumulation: any particle order gives the same bits (the REDG path cannot promise that)"""
    N, L = 64, 200.
    pos = _particles(300000, [L] * 3, "f4", outside=False)
    pm = _pm(N, L, "f8")
    a = pm.paint(pos, resampler="tsc", method='tiled').numpy()
    perm = np.random.RandomState(1).permutation(len(pos))
    b = pm.paint(pos[perm], resampler="tsc", method='tiled').numpy()
    order = np.lexsort((pos[:, 2], pos[:, 1], pos[:, 0]))
    c = pm.paint(pos[order], resampler="tsc", method='tiled').numpy()
    assert np.array_equal(a, b) and np.array_equal(a, c)


def test_paint_tiled_interlaced_hold_and_shift(cuda):
    from nbodykit_b200.pmesh.pm import RealField
    N, L = [32, 32, 64], 100.
    pos = _particles(150000, [L] * 3, "f4")
    mass = np.random.RandomState(5).uniform(0.1, 1.0, size=len(pos)).astype("f4")
    pm = _pm(N, L, "f8")
    r1, r2 = RealField(pm), RealField(pm)
    r1[...] = 1.0; r2[...] = 2.0          # hold semantics: accumulate into what is there
    pm.paint_interlaced(pos, mass, "tsc", r1, r2, method='tiled')
    w1 = 1.0 + po.paint(pos, mass, N, L, "tsc", 0.0)
    w2 = 2.0 + po.paint(pos, mass, N, L, "tsc", 0.5)
    np.testing.assert_allclose(r1.numpy(), w1, rtol=0, atol=1e-7 * w1.max())
    np.testing.assert_allclose(r2.numpy(), w2, rtol=0, atol=1e-7 * w2.max())
    out = pm.paint(pos, mass=mass, resampler="cic", transform=pm.affine.shift(0.5), method='tiled')
    w = po.paint(pos, mass, N, L, "cic", 0.5)
    np.testing.assert_allclose(out.numpy(), w, rtol=0, atol=1e-7 * w.max())


def test_paint_tiled_slab_ghosts(cuda):
    """x slabs: ghost particles (leftmost cell below the slab) contribute only their in-slab planes"""
    import ctypes
    import torch
    from nbodykit_b200 import _lib
    N, L = [64, 32, 32], [64., 32., 32.]
    pos = _particles(120000, L, "f4")
    full = po.paint(pos, None, N, L, "tsc")
    p = torch.from_numpy(pos).cuda()
    Lb = _lib.lib()
    for x0, xn in [(0, 16), (16, 16), (48, 16), (8, 40)]:
        for shift in (0.0, 0.5):
            want = full if shift == 0.0 else po.paint(pos, None, N, L, "tsc", 0.5)
            mesh = torch.full((xn, 32, 32), 3.0, dtype=torch.float64, device="cuda")   # clear=1 must wipe this
            nb = Lb.nbk_paint_tiled_workspace(len(pos), 4, 0, _lib.iarr(N), xn)
            work = torch.empty(nb, dtype=torch.uint8, device="cuda")
            _lib.check(Lb.nbk_paint_tiled(ctypes.c_void_p(p.data_ptr()), 4, len(pos), None, 8, 3, shift, _lib.darr(L),
                                          _lib.iarr(N), x0, xn, ctypes.c_void_p(mesh.data_ptr()), None, 8,
                                          ctypes.c_void_p(work.data_ptr()), nb, 1, None))
            torch.cuda.synchronize()
            np.testing.assert_allclose(mesh.cpu().numpy(), want[x0:x0 + xn], rtol=0, atol=1e-7 * want.max())


def test_paint_tiled_clustered_and_empty_tiles(cuda):
    """all particles inside two cells (one hot tile, thousands of empty ones) + a tile on the periodic seam"""
    N, L = 64, 64.
    rng = np.random.RandomState(8)
    pos = np.concatenate([rng.uniform(10.0, 11.0, size=(100000, 3)), rng.uniform(63.0, 64.0, size=(100000, 3))]).astype("f4")
    pm = _pm(N, L, "f4")
    got = pm.paint(pos, resampler="cic", method='tiled').numpy()
    want = po.paint(pos, None, N, L, "cic")
    np.testing.assert_allclose(got, want, rtol=0, atol=3e-7 * want.max())
    assert abs(got.sum(dtype="f8") - len(pos)) < 1e-2


def test_paint_tiled_many_tiles_uses_global_bucketing(cuda):
    """more tiles than a shared-memory histogram holds (> 51200): the bucketing falls back to global counters;
    checked against the direct REDG scatter on the same particles"""
    N, L = [1024, 1024, 256], [1000., 1000., 250.]
    pos = _particles(3000000, L, "f4")
    pm = _pm(N, L, "f4")
    a = pm.paint(pos, resampler="cic", method='tiled')
    b = pm.paint(pos, resampler="cic", method='direct')
    d = (a.value - b.value).abs().max().item()
    assert d <= 2e-5 * b.value.abs().max().item()
    assert abs(a.csum() - len(pos)) < 2.0 and abs(b.csum() - len(pos)) < 2.0


def test_paint_auto_dispatch_matches(cuda):
    """the default dispatch (tiled for dense catalogues, direct otherwise) is transparent"""
    N, L = 32, 50.
    pm = _pm(N, L, "f8")
    for n in (5000, 200000):
        pos = _particles(n, [L] * 3, "f4")
        a = pm.paint(pos, resampler="cic").numpy()
        w = po.paint(pos, None, N, L, "cic")
        np.testing.assert_allclose(a, w, rtol=0, atol=1e-7 * w.max())


def test_power_bin_fused_compensation_equals_two_pass(cuda):
    """nbk_power_bin(comp1, comp2) == nbk_compensate on each field followed by nbk_power_bin"""
    from nbodykit_b200.algorithms.fftpower import project_to_basis_device
    from nbodykit_b200.pmesh.pm import ComplexField
    N, L = [16, 32, 16], [100., 200., 100.]
    rng = np.random.RandomState(21)
    shape = (N[0], N[1], N[2] // 2 + 1)
    a = rng.standard_normal(shape) + 1j * rng.standard_normal(shape)
    b = rng.standard_normal(shape) + 1j * rng.standard_normal(shape)
    pm = _pm(N, L, "f8")
    dk = 2 * np.pi / 100.
    edges = [np.arange(0., np.pi * 16 / 200. + dk / 2, dk), np.linspace(-1, 1, 4)]
    for n1, n2 in [("CompensateCICShotnoise", "CompensateCICShotnoise"), ("CompensateTSC", "CompensatePCSShotnoise")]:
        f1, f2 = ComplexField(pm), ComplexField(pm)
        f1[...] = a; f2[...] = b
        fused = project_to_basis_device(f1, edges, poles=[0, 2], is_p3d=False, second=f2, volume=3.0,
                                        compensation=(n1, n2))
        f1.compensate(n1); f2.compensate(n2)
        two = project_to_basis_device(f1, edges, poles=[0, 2], is_p3d=False, second=f2, volume=3.0)
        assert np.array_equal(fused[0][3], two[0][3])
        np.testing.assert_allclose(np.nan_to_num(fused[0][2]), np.nan_to_num(two[0][2]), rtol=1e-12)
        np.testing.assert_allclose(np.nan_to_num(fused[1][1]), np.nan_to_num(two[1][1]), rtol=1e-11, atol=1e-12)
    # auto power: the same transfer function applies to both factors
    f1 = ComplexField(pm); f1[...] = a
    fused = project_to_basis_device(f1, edges, is_p3d=False, volume=1.0, compensation=("CompensateTSCShotnoise", None))
    f1.compensate("CompensateTSCShotnoise")
    two = project_to_basis_device(f1, edges, is_p3d=False, volume=1.0)
    np.testing.assert_allclose(np.nan_to_num(fused[0][2]), np.nan_to_num(two[0][2]), rtol=1e-12)


def test_r2c_extra_scale(cuda):
    from nbodykit_b200.pmesh.pm import RealField
    real = np.random.RandomState(6).standard_normal((16, 16, 16))
    pm = _pm(16, 1.0, "f8")
    f = RealField(pm)
    f[...] = real
    np.testing.assert_allclose(f.r2c(scale=2.5).numpy(), 2.5 * f.r2c().numpy(), rtol=1e-14)


def test_route_kernels_vs_numpy(cuda):
    """nbk_route_count / nbk_route_scatter: destination bitmask, counts and compacted send segments"""
    import ctypes
    import torch
    from nbodykit_b200 import _lib
    N, L, P, rank = [64, 16, 16], [128., 16., 16.], 4, 1
    rng = np.random.RandomState(31)
    pos = rng.uniform(-40, 170, size=(50000, 3)).astype("f4")
    mass = rng.uniform(size=len(pos))
    Lb = _lib.lib()
    p = torch.from_numpy(pos).cuda(); m = torch.from_numpy(mass).cuda()
    for smoothing in (1.0, 1.5, 3.0):
        ghosts = torch.empty(len(pos), dtype=torch.int64, device="cuda")
        counts = torch.zeros(P + 1, dtype=torch.int64, device="cuda")
        _lib.check(Lb.nbk_route_count(ctypes.c_void_p(p.data_ptr()), 4, len(pos), smoothing, _lib.darr(L), _lib.iarr(N), P, rank,
                                      ctypes.c_void_p(counts.data_ptr()), ctypes.c_void_p(ghosts.data_ptr()), None))
        gx = pos[:, 0].astype("f8") * (N[0] / L[0])
        want = np.zeros(len(pos), dtype="i8")
        for c in range(-4, 5):
            cell = np.floor(gx + c * 1.0)           # enumerate integer cells in [floor(gx-s), floor(gx+s)]
        lo, hi = np.floor(gx - smoothing).astype("i8"), np.floor(gx + smoothing).astype("i8")
        for off in range(0, 8):
            cell = lo + off
            ok = cell <= hi
            r = (cell % N[0]) // (N[0] // P)
            want |= np.where(ok, 1 << r, 0)
        want &= ~(1 << rank)
        nl = int(counts[P].item())
        ent = ghosts[:nl].cpu().numpy()
        got = np.zeros(len(pos), dtype="i8")
        assert len(np.unique(ent & 0xffffffff)) == nl                 # every travelling particle listed once
        got[ent & 0xffffffff] = ent >> 32
        assert np.array_equal(got, want) and nl == int((want != 0).sum())
        cnt = [int(((want >> r) & 1).sum()) for r in range(P)]
        assert counts[:P].cpu().tolist() == cnt and cnt[rank] == 0
        off = torch.tensor([0] + list(np.cumsum(cnt)[:-1]), dtype=torch.int64, device="cuda")
        cur = torch.zeros(P, dtype=torch.int64, device="cuda")
        spos = torch.empty((sum(cnt), 3), dtype=torch.float32, device="cuda")
        smass = torch.empty(sum(cnt), dtype=torch.float64, device="cuda")
        sidx = torch.empty(sum(cnt), dtype=torch.int64, device="cuda")
        _lib.check(Lb.nbk_route_scatter(ctypes.c_void_p(p.data_ptr()), 4, ctypes.c_void_p(m.data_ptr()), 8,
                                        ctypes.c_void_p(ghosts.data_ptr()), nl, P, ctypes.c_void_p(off.data_ptr()),
                                        ctypes.c_void_p(cur.data_ptr()), ctypes.c_void_p(spos.data_ptr()),
                                        ctypes.c_void_p(smass.data_ptr()), ctypes.c_void_p(sidx.data_ptr()), None))
        torch.cuda.synchronize()
        sp, sm = spos.cpu().numpy(), smass.cpu().numpy()
        # the source-row column points back at the rows that were copied
        assert np.array_equal(pos[sidx.cpu().numpy()], sp)
        start = 0
        for r in range(P):
            sel = ((want >> r) & 1).astype(bool)
            seg = slice(start, start + cnt[r])
            # same multiset of (x, y, z, mass) rows, any order
            a = np.concatenate([sp[seg].astype("f8"), sm[seg][:, None]], axis=1)
            b = np.concatenate([pos[sel].astype("f8"), mass[sel][:, None]], axis=1)
            assert np.array_equal(a[np.lexsort(a.T)], b[np.lexsort(b.T)])
            start += cnt[r]


# chunks = 1 is the whole slab in one part (the c2r exchange).  The line lengths cover every pack kernel: N < 64 (shared
# memory), N = 64 and 128 (register I/O), N = 256, 512 and 1024 (TMA; f4 with Nz/2+1 = 3 columns takes the misaligned
# register-I/O fallback)
@pytest.mark.parametrize("shape,chunks", [((16, 32, 8), 4), ((8, 256, 16), 3), ((256, 64, 4), 5), ((128, 64, 32), 3),
                                          ((16, 32, 8), 1), ((64, 128, 8), 1), ((128, 64, 32), 1), ((4, 256, 8), 1),
                                          ((256, 512, 4), 1), ((2, 1024, 16), 1)])
@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_fft_pack_push_range_two_virtual_ranks(cuda, dtype, shape, chunks):
    """the slab exchange of the distributed r2c / c2r: nbk_fft_lines_pack_range (y pass of a part of the slab into the
    send blocks) + nbk_slab_push_range (strided bulk copies of that part into the owners' transposed fields), part by part,
    must give the transposed field of the one-shot y pass -- two virtual ranks on one GPU (the peers are two buffers of
    this device), uneven last part included"""
    import ctypes
    import torch
    from nbodykit_b200 import _lib
    (Nx, Ny, Nz), P = shape, 2
    Nzc = Nz // 2 + 1
    rng = np.random.RandomState(23)
    real = rng.standard_normal((Nx, Ny, Nz)).astype(dtype)
    want = np.fft.rfftn(real.astype("f8")) / real.size
    cdt = torch.complex64 if dtype == "f4" else torch.complex128
    code = 4 if dtype == "f4" else 8
    Lb = _lib.lib()
    x_n, y_n = Nx // P, Ny // P
    stage = [torch.zeros((y_n, Nx, Nzc), dtype=cdt, device="cuda") for _ in range(P)]
    ptrs = (ctypes.c_void_p * P)(*[t.data_ptr() for t in stage])
    per = (x_n + chunks - 1) // chunks
    for r in range(P):
        slab = torch.from_numpy(real[r * x_n:(r + 1) * x_n].copy()).cuda()
        work = torch.empty((x_n, Ny, Nzc), dtype=cdt, device="cuda")
        send = torch.zeros((P, y_n, x_n, Nzc), dtype=cdt, device="cuda")
        _lib.check(Lb.nbk_fft_z_forward(ctypes.c_void_p(slab.data_ptr()), ctypes.c_void_p(work.data_ptr()), code, x_n * Ny, Nz, None))
        for c in range(chunks):
            o0 = c * per
            oc = min(per, x_n - o0)
            if oc <= 0:
                break
            _lib.check(Lb.nbk_fft_lines_pack_range(ctypes.c_void_p(work.data_ptr()), ctypes.c_void_p(send.data_ptr()), code, Ny, Nzc,
                                                   x_n, o0, oc, P, 0, 1.0, None))
            _lib.check(Lb.nbk_slab_push_range(ctypes.c_void_p(send.data_ptr()), ptrs, code, y_n, x_n, Nzc, r * x_n, o0, oc, P, r, None))
    torch.cuda.synchronize()
    tol = 1e-13 if dtype == "f8" else 2e-6
    for r in range(P):
        out = torch.empty_like(stage[r])
        _lib.check(Lb.nbk_fft_lines_oop(ctypes.c_void_p(stage[r].data_ptr()), ctypes.c_void_p(out.data_ptr()), code, Nx, Nzc, Nzc,
                                        y_n, Nx * Nzc, 0, 1.0 / real.size, None))
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        ref = np.transpose(want[:, r * y_n:(r + 1) * y_n, :], (1, 0, 2))
        assert np.abs(got - ref).max() <= tol * np.sqrt((np.abs(want) ** 2).mean()) * 10
