"""
The run plan of the tiled paint (NBK_PAINT_BUCKET=runs): bucketing runs of consecutive same-tile particles and
rebuilding each particle's record in the tile pass must give the mesh of the record plans BIT FOR BIT on f8 meshes (same
records, fixed-point accumulation, exact f8 sums of the halo shares), on every window, position dtype, mass kind,
particle order, slab and write-back.  On f4 meshes the halo shares of neighbouring tiles are added in float32 in an order
that depends on timing, in every plan, so f4 meshes agree to float32 rounding.  The probe's choice of plan is read back
from the workspace header through the C ABI.
"""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N3, L3 = [64, 48, 64], [128., 96., 128.]        # power-of-two N/L on x and z, not on y: both record paths
HDR_MODE_BYTE = 8                                 # workspace header word 2
MODES = {0: "scattered", 1: "coherent", 2: "runs"}


def _pm(N, L, dtype):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.pmesh.pm import ParticleMesh
    return ParticleMesh(BoxSize=L, Nmesh=N, dtype=dtype, comm=SelfComm())


def generator_catalogue(N, L, dtype="f4", per=8, seed=3):
    """a mock generator's output: generator cells of two mesh cells in x, y, z order, each emitting its particles
    together, jittered inside the cell and moved by a smooth displacement (~0.7 generator cells)"""
    rng = np.random.RandomState(seed)
    ng = [n // 2 for n in N]
    cs = np.asarray(L, dtype="f8") / ng
    cells = np.indices(ng).reshape(3, -1).T
    counts = rng.poisson(per, size=len(cells))
    c = np.repeat(cells, counts, axis=0).astype("f8")
    disp = 0.7 * cs * np.sin(2 * np.pi * (c[:, [1, 2, 0]] + 0.5) / np.asarray(ng)[[1, 2, 0]] + np.arange(3))
    pos = (c + rng.uniform(0, 1, size=c.shape)) * cs + disp
    return np.mod(pos, np.asarray(L)).astype(dtype)


def orders(pos):
    return {"generator": np.arange(len(pos)),
            "x-sorted": np.argsort(pos[:, 0], kind="stable"),
            "random": np.random.RandomState(4).permutation(len(pos))}


def masses(kind, n, seed=11):
    rng = np.random.RandomState(seed)
    if kind == "none":
        return None
    if kind == "positive":
        return rng.uniform(0.1, 2.0, size=n)
    return rng.uniform(-1.0, 2.0, size=n).astype("f4")          # signed, float32 masses


def paint(pm, pos, mass, resampler, plan, monkeypatch, **kw):
    monkeypatch.setenv("NBK_PAINT_BUCKET", plan)
    return pm.paint(pos, mass=1.0 if mass is None else mass, resampler=resampler, method="tiled", **kw).numpy()


def assert_runs_equal_scattered(pm, pos, mass, resampler, monkeypatch, what, **kw):
    a = paint(pm, pos, mass, resampler, "runs", monkeypatch, **kw)
    b = paint(pm, pos, mass, resampler, "scattered", monkeypatch, **kw)
    if b.dtype == np.float64:
        assert np.array_equal(a, b), what
    else:
        np.testing.assert_allclose(a, b, rtol=0, atol=1e-6 * np.abs(b).max(), err_msg=what)
    return a


def abi_paint(pos_t, n, window, N, L, x0, xn, shift, mesh, mass_t=None, mass_code=8):
    """nbk_paint_tiled through ctypes; returns the plan the workspace header records"""
    import torch
    from nbodykit_b200 import _lib
    Lb = _lib.lib()
    pcode = 4 if pos_t.dtype == torch.float32 else 8
    mcode = 8 if mesh.dtype == torch.float64 else 4
    nb = Lb.nbk_paint_tiled_workspace(n, pcode, mass_code if mass_t is not None else 0, _lib.iarr(N), xn)
    work = torch.empty(nb, dtype=torch.uint8, device="cuda")
    _lib.check(Lb.nbk_paint_tiled(ctypes.c_void_p(pos_t.data_ptr()), pcode, n,
                                  ctypes.c_void_p(mass_t.data_ptr()) if mass_t is not None else None, mass_code, window,
                                  shift, _lib.darr(L), _lib.iarr(N), x0, xn, ctypes.c_void_p(mesh.data_ptr()), None, mcode,
                                  ctypes.c_void_p(work.data_ptr()), nb, 1, None))
    torch.cuda.synchronize()
    return MODES[int(work[HDR_MODE_BYTE:HDR_MODE_BYTE + 4].cpu().numpy().view(np.uint32)[0])]


@pytest.mark.parametrize("resampler", ["nnb", "cic", "tsc", "pcs"])
@pytest.mark.parametrize("pos_dtype", ["f4", "f8"])
@pytest.mark.parametrize("mesh_dtype", ["f4", "f8"])
def test_runs_match_scattered(cuda, monkeypatch, resampler, pos_dtype, mesh_dtype):
    """every window, position and mesh dtype, mass kind and order (x-sorted: fragmented runs; random: runs of one)"""
    pos = generator_catalogue(N3, L3, pos_dtype)
    pm = _pm(N3, L3, mesh_dtype)
    for mkind in ("none", "positive", "signed"):
        mass = masses(mkind, len(pos))
        for oname, idx in orders(pos).items():
            m = mass[idx] if mass is not None else None
            assert_runs_equal_scattered(pm, pos[idx], m, resampler, monkeypatch, "%s %s" % (mkind, oname))


def test_runs_odd_count_unaligned_positions(cuda, monkeypatch):
    """n not a multiple of 4 and a position pointer 4 bytes off a 16-byte boundary (the scalar quad loads)"""
    import torch
    pos = generator_catalogue(N3, L3, "f4")[:100003]
    buf = torch.zeros(3 * len(pos) + 1, dtype=torch.float32, device="cuda")
    buf[1:] = torch.from_numpy(pos.ravel()).cuda()
    p = buf[1:].view(len(pos), 3)
    assert p.data_ptr() % 16 != 0
    pm = _pm(N3, L3, "f8")
    for resampler in ("cic", "tsc"):
        got = assert_runs_equal_scattered(pm, p, None, resampler, monkeypatch, resampler)
        assert abs(got.sum(dtype="f8") - len(pos)) < 1e-6 * len(pos)


def test_runs_one_cell_catalogue(cuda, monkeypatch):
    """every particle in one cell: runs capped at 128 particles, one dense tile"""
    pos = np.random.RandomState(2).uniform(20.0, 22.0, size=(200001, 3)).astype("f4")
    pm = _pm(N3, L3, "f8")
    for resampler in ("cic", "pcs"):
        assert_runs_equal_scattered(pm, pos, None, resampler, monkeypatch, resampler)
    mass = masses("signed", len(pos))
    assert_runs_equal_scattered(pm, pos, mass, "tsc", monkeypatch, "signed")


def test_runs_cell_and_tile_boundaries(cuda, monkeypatch):
    """particles exactly on cell and tile faces, at x = L, and the mesh edges, in cell order"""
    rng = np.random.RandomState(5)
    cs = np.asarray(L3) / np.asarray(N3)
    pos = generator_catalogue(N3, L3, "f8", per=4)
    k = rng.randint(0, 3, size=pos.shape)                 # 0: leave, 1: snap to a cell face, 2: snap to a tile face
    cell = np.floor(pos / cs)
    tile = np.floor(pos / (16 * cs)) * 16
    pos = np.where(k == 1, cell * cs, np.where(k == 2, tile * cs, pos))
    pos[::97, 0] = L3[0]
    pos[1::97] = np.asarray(L3)
    pos[2::97] = 0.0
    pm = _pm(N3, L3, "f8")
    for pdt in ("f8", "f4"):
        for resampler in ("nnb", "cic", "tsc", "pcs"):
            assert_runs_equal_scattered(pm, pos.astype(pdt), None, resampler, monkeypatch, "%s %s" % (pdt, resampler))


def test_runs_out_of_window_tiles(cuda, monkeypatch):
    """512^3: 32768 tiles, more than the coherent window holds -- in random order nearly every run's tile lies outside
    its chunk's window (global counters and cursors); NBK_PAINT_W=16 does the same to the generator order"""
    N, L = [512] * 3, [1024.] * 3
    pos = generator_catalogue([128] * 3, L, "f4", per=4)
    pm = _pm(N, L, "f8")
    for oname, idx in orders(pos).items():
        assert_runs_equal_scattered(pm, pos[idx], None, "cic", monkeypatch, oname)
    monkeypatch.setenv("NBK_PAINT_W", "16")
    assert_runs_equal_scattered(pm, pos, None, "cic", monkeypatch, "window of 16 tiles")


def test_runs_interlaced_hold_and_shift(cuda, monkeypatch):
    """the interlaced pair (two tile passes over one set of runs), hold=True (TMA reduce-add) and shift 0.5"""
    from nbodykit_b200.pmesh.pm import RealField
    pos = generator_catalogue(N3, L3, "f4")
    mass = masses("positive", len(pos)).astype("f4")
    pm = _pm(N3, L3, "f8")
    got = {}
    for plan in ("runs", "scattered"):
        monkeypatch.setenv("NBK_PAINT_BUCKET", plan)
        r1, r2 = RealField(pm), RealField(pm)
        r1[...] = 1.0
        r2[...] = 2.0
        pm.paint_interlaced(pos, mass, "tsc", r1, r2, method="tiled", hold=True)
        r3, r4 = RealField(pm), RealField(pm)
        pm.paint_interlaced(pos, None, "cic", r3, r4, method="tiled", hold=False)
        s = pm.paint(pos, mass=mass, resampler="pcs", transform=pm.affine.shift(0.5), method="tiled")
        h = RealField(pm)
        h[...] = 0.5
        pm.paint(pos, resampler="cic", hold=True, out=h, method="tiled")
        got[plan] = [r1.numpy(), r2.numpy(), r3.numpy(), r4.numpy(), s.numpy(), h.numpy()]
    for i, (a, b) in enumerate(zip(got["runs"], got["scattered"])):
        assert np.array_equal(a, b), i


def test_runs_slab_ghosts(cuda, monkeypatch):
    """x slabs through the C ABI: ghost particles (leftmost cell below the slab) paint only their in-slab planes"""
    import torch
    N, L = [64, 32, 32], [64., 32., 32.]
    pos = generator_catalogue(N, L, "f4")
    p = torch.from_numpy(pos).cuda()
    mass = torch.from_numpy(masses("signed", len(pos)).astype("f8")).cuda()
    for x0, xn in [(0, 16), (16, 16), (48, 16), (8, 40)]:
        for shift in (0.0, 0.5):
            for m in (None, mass):
                got = {}
                for plan in ("runs", "scattered"):
                    monkeypatch.setenv("NBK_PAINT_BUCKET", plan)
                    mesh = torch.full((xn, 32, 32), 3.0, dtype=torch.float64, device="cuda")
                    assert abi_paint(p, len(pos), 3, N, L, x0, xn, shift, mesh, m) == plan
                    got[plan] = mesh.cpu().numpy()
                assert np.array_equal(got["runs"], got["scattered"]), (x0, xn, shift, m is None)


def test_probe_picks_plan(cuda, monkeypatch):
    """without NBK_PAINT_BUCKET the probe picks runs for the generator order, coherent for the x-sorted order (same
    planes, few equal-tile neighbours) and scattered for a random order -- and every plan paints the same mesh"""
    import torch
    monkeypatch.delenv("NBK_PAINT_BUCKET", raising=False)
    pos = generator_catalogue(N3, L3, "f4")
    want = {"generator": "runs", "x-sorted": "coherent", "random": "scattered"}
    meshes = []
    for oname, idx in orders(pos).items():
        p = torch.from_numpy(np.ascontiguousarray(pos[idx])).cuda()
        mesh = torch.zeros(N3, dtype=torch.float64, device="cuda")
        assert abi_paint(p, len(pos), 2, N3, L3, 0, N3[0], 0.0, mesh) == want[oname], oname
        meshes.append(mesh.cpu().numpy())
    assert np.array_equal(meshes[0], meshes[1]) and np.array_equal(meshes[0], meshes[2])
