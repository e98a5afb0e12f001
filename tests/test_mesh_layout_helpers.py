"""
CPU checks of the helpers behind tests/test_gpu_mesh_layouts.py (oracle/mesh_layouts.py): the slab split and
reassembly, the boundary-position generator (do its positions reach the float32 margin and both sides of every
targeted boundary?), the fixed-point scale and the per-cell deposit bound of the tiled paint.
"""
import numpy as np
import pytest

from oracle import mesh_layouts as ml
from oracle import pmesh_oracle as po

PAINT_N = (48, 64, 80)
BOXES = {"margin": (100., 3.3, 7000.), "pow2": (96., 64., 40.)}


@pytest.mark.parametrize("shape", [(45, 21, 18), (44, 52, 19), (48, 36, 9)])
def test_slab_split_and_join(shape):
    a = np.random.RandomState(0).standard_normal(shape)
    for P in ml.rank_counts(shape[1]):
        parts = ml.split_transposed(a, P)
        assert len(parts) == P
        for r, p in enumerate(parts):
            assert p.flags.c_contiguous and p.shape == (shape[1] // P, shape[0], shape[2])
            y_n = shape[1] // P
            assert np.array_equal(p[1], a[:, r * y_n + 1, :])
        assert np.array_equal(ml.join_transposed(parts), a)
    for P in ml.rank_counts(shape[0]):
        parts = ml.split_x(a, P)
        assert all(p.flags.c_contiguous for p in parts)
        assert np.array_equal(np.concatenate(parts), a)
    assert ml.rank_counts(21) == [3] and ml.rank_counts(52) == [2, 4] and ml.rank_counts(36) == [2, 3, 4]


def _float32_cell(x, n, l, res):
    """the leftmost cell in float32 arithmetic alone: floor(fl32(fl32(x) * fl32(N/L)) + A) + B"""
    g = (np.asarray(x, dtype=np.float32) * np.float32(float(n) / float(l))).astype("f8")
    return np.floor(g + ml.WIN_A[res]).astype("i8") + ml.WIN_B[res]


@pytest.mark.parametrize("box", sorted(BOXES))
@pytest.mark.parametrize("dtype", ["f4", "f8"])
@pytest.mark.parametrize("res", ["nnb", "cic", "tsc", "pcs"])
def test_boundary_positions_reach_the_boundaries(box, dtype, res):
    N, L = PAINT_N, BOXES[box]
    pos, nsp = ml.boundary_positions(N, L, dtype, seed=5)
    assert pos.dtype == np.dtype(dtype) and len(pos) >= 100000 and 0 < nsp < len(pos)
    for d in range(3):
        vals = ml.boundary_values(N, L, dtype)[d]
        assert np.isin(vals, pos[:nsp, d]).all()
        n, l = N[d], L[d]
        g = vals.astype("f8") * (float(n) / float(l))
        cell = ml.exact_cell(vals, n, l, res)
        # both sides of every targeted boundary k - A (k in {0, 1, N/2, N-1, N}), in the exact f8 arithmetic
        for k in (0, 1, n // 2, n - 1, n):
            near = np.abs(g + ml.WIN_A[res] - k) < 1e-3
            assert (cell[near] == k + ml.WIN_B[res]).any() and (cell[near] == k - 1 + ml.WIN_B[res]).any(), (d, k)
        # |g| just below and just above the 2^22 limit of the float32 record / tile paths, on both sides of zero
        for s in (1.0, -1.0):
            assert ((s * g < 4194304.0) & (s * g > 4194300.0)).any() and ((s * g >= 4194304.0) & (s * g < 4194308.0)).any()
        assert (np.abs(vals.astype("f8")) > 900 * l).any() and (vals == l).any()
        assert (np.signbit(vals) & (vals == 0)).any()                 # -0.0
        if dtype == "f4" and box == "margin":
            # the float32 tile id is not decisive for some of them: the count pass recomputes those in f8 ...
            assert ml.fast_tile_needs_f8(vals, n, l, res).any()
            # ... and float32 arithmetic alone puts some in another cell than the f8 contract
            inbox = np.abs(g) < 4194304.0
            assert (_float32_cell(vals[inbox], n, l, res) != cell[inbox]).any()
        if dtype == "f4" and box == "pow2":
            # N/L a power of two: x * N/L is exact in float32 (the premise of the shortcut), denormals aside
            g32 = vals * np.float32(float(n) / float(l))
            normal = np.abs(vals) > 1e-30
            assert np.array_equal(g32[normal].astype("f8"), g[normal])
            # the two float32 traps of the record / tile arithmetic are among them: g + 1/2 rounded in float32 reaches
            # the next integer (g = 1/2 - 2^-25) ...
            if ml.WIN_A[res]:
                assert (np.floor(g32 + np.float32(0.5)) != np.floor(g + 0.5)).any()
            # ... and g - floor(g) rounds to 1.0 (g in (-2^-25, 0))
            assert ((g32 - np.floor(g32)).astype(np.float32) == np.float32(1.0)).any()


def test_fixed_point_scale():
    assert ml.fixed_point_scale(None) == 1.0
    assert ml.fixed_point_scale(np.zeros(5)) == 1.0
    assert ml.fixed_point_scale(np.array([0.5, 7.5])) == 8.0
    assert ml.fixed_point_scale(np.array([8.0])) == 16.0                  # the 1.0000001f margin lifts 2^k to the next
    assert ml.fixed_point_scale(np.array([np.nextafter(np.float32(8), np.float32(0))])) == 16.0
    assert ml.fixed_point_scale(np.array([-3.0, 1.0])) == 4.0
    rng = np.random.RandomState(1)
    for _ in range(200):
        m = rng.standard_normal(10) * 10.0 ** rng.uniform(-8, 8)
        M = ml.fixed_point_scale(m)
        assert np.abs(m).max() < M <= 4 * np.abs(m).max()


@pytest.mark.parametrize("res", ["nnb", "cic", "tsc", "pcs"])
def test_deposit_bound_and_nnb_fixed_point(res):
    N, L = PAINT_N, BOXES["margin"]
    pos, _ = ml.boundary_positions(N, L, "f4", n_total=20000, repeat=1, seed=2)
    m = np.random.RandomState(3).uniform(-2, 5, size=len(pos))
    bound, cnt = ml.deposit_bound(pos, m, N, L, res)
    sup = po.SUPPORT[res]
    assert cnt.sum() == len(pos) * sup ** 3
    M = ml.fixed_point_scale(m)
    assert M == 8.0
    assert (bound >= cnt * M * 2.0 ** -32).all() and bound.max() < 1e-6 * M * cnt.max()
    if res == "nnb":
        assert np.array_equal(cnt, po.paint(pos, None, N, L, "nnb"))
        assert np.array_equal(ml.nnb_fixed_point(pos, None, N, L), po.paint(pos, None, N, L, "nnb"))
        fp = ml.nnb_fixed_point(pos, m, N, L)
        want = po.paint(pos, m, N, L, "nnb")
        assert (np.abs(fp - want) <= bound).all() and not np.array_equal(fp, want)


def test_project_sums_anti_matches_full_mesh():
    """the anti-Hermitian fold of the compressed half equals binning every mode of the full mesh (odd sides: every
    mirror is stored with the negated label); Nmu = 1 with the mu = 1 column folded, since a mirror has the opposite mu"""
    N, L = (15, 9, 11), (10., 12., 9.)
    rng = np.random.RandomState(4)
    r = rng.standard_normal(N)
    full = 1j * np.fft.fftn(r)
    comp = 1j * np.fft.rfftn(r)
    edges = [np.arange(0., 3.0, 0.6), np.linspace(-1, 1, 2)]
    a = ml.project_sums_anti(comp, po.k_coords(N, L, "f8"), edges, [0, 0, 1], [1, 2, 3])
    b = po.project_sums(full, ml.k_coords(N, L, "f8", fullz=True), edges, [0, 0, 1], [1, 2, 3], hermitian_symmetric=False)
    for s in (a, b):
        s[3][:, 1] += s[3][:, 2]
        s[2][..., 1] += s[2][..., 2]
    assert np.array_equal(a[3][:, :2], b[3][:, :2])
    np.testing.assert_allclose(a[2][..., :2], b[2][..., :2], rtol=1e-12, atol=1e-12 * np.abs(b[2]).max())
    # odd sides: the mirror direction is -khat everywhere
    khat, mhat = ml.mirror_dirs(N, L)
    for d in range(3):
        np.testing.assert_array_equal(mhat[d], -khat[d])


# ---- the slab-edge generator of tests/test_gpu_slab_route.py --------------------------------------------------------
ROUTE_GEOMS = [((48, 32, 32), 3), ((40, 32, 32), 8), ((32, 32, 32), 8), ((64, 16, 16), 32)]
SMOOTHINGS = (0.5, 1.0, 1.5, 2.0, 2.5, 3.0, 4.0)


@pytest.mark.parametrize("NP", ROUTE_GEOMS, ids=lambda g: "%s-P%d" % g if isinstance(g, tuple) else str(g))
@pytest.mark.parametrize("lx", [100., 24.])
@pytest.mark.parametrize("dtype", ["f4", "f8"])
def test_slab_edge_positions_reach_both_sides(NP, lx, dtype):
    """every slab-edge target b + d is straddled in exact f8 grid units, every float32 rejection edge in the route's
    float32 arithmetic, and the seam images 1 .. 3 box lengths out are present"""
    N, P = NP
    Nx = N[0]
    L = (lx, 30., 30.)
    pos, n_edge = ml.slab_edge_positions(N, L, P, SMOOTHINGS, dtype)
    assert pos.dtype == np.dtype(dtype) and n_edge > 0
    x = pos[:n_edge, 0]
    g = x.astype("f8") * (Nx / lx)
    for t in ml.slab_edge_targets(Nx, P, SMOOTHINGS):
        near = np.abs(g - t) < 1e-3
        assert (g[near] < t).any() and (g[near] >= t).any(), "target %g" % t
    g32 = x.astype(np.float32) * np.float32(Nx / lx)
    for s in SMOOTHINGS:
        for lo, hi in ml.route_reject_edges(Nx, P, s):
            for e in (lo, hi):
                near = np.abs(g32.astype("f8") - float(e)) < 1e-3
                assert (g32[near] > e).any() and (g32[near] <= e).any(), "edge %g (s=%g)" % (e, s)
    for j in (-3, -1, 1, 3):
        assert (np.abs(g - j * Nx) < 1e-3).any()
    assert (np.signbit(x) & (x == 0)).any() and (~np.signbit(x) & (x == 0)).any()


def test_route_margin_and_stencil_ranks():
    assert ml.route_margin(1024) == np.float32(1e-3) + np.float32(4e-7) * np.float32(1024)
    N, L, P = (16, 4, 4), (16., 4., 4.), 4                      # x_n = 4, one cell per unit length
    x = np.array([3.5, 3.99, 0.2, 15.7, 7.5, 8.0])
    pos = np.stack([x, np.ones_like(x), np.ones_like(x)], axis=1)
    # cic: cells floor(g), floor(g) + 1; shift 0.5 moves both up by one when frac(g) >= 1/2
    assert ml.stencil_ranks(pos, N, L, P, "cic", [0.0]).tolist() == [0b11, 0b11, 0b1, 0b1001, 0b110, 0b100]
    assert ml.stencil_ranks(pos, N, L, P, "cic", [0.0, 0.5]).tolist() == [0b11, 0b11, 0b1, 0b1001, 0b110, 0b100]
    # nnb: the nearest cell floor(g + 1/2); pcs: floor(g) - 1 .. floor(g) + 2
    assert ml.stencil_ranks(pos, N, L, P, "nnb", [0.0]).tolist() == [0b10, 0b10, 0b1, 0b1, 0b100, 0b100]
    assert ml.stencil_ranks(pos, N, L, P, "pcs", [0.0]).tolist() == [0b11, 0b11, 0b1001, 0b1001, 0b110, 0b110]
