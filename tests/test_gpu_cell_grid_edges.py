"""The cell grid shared by FOF, the pair counts and the 3PCF (the keys of csrc/fof.cu, the key sort and compaction, the
stencil of csrc/pc_cells.cuh) at its edges, against the CPU restatements in oracle/: box sides that float32 cannot
hold (a row wrapped onto L_f4 != L), cell counts at their ceil / floor boundaries and at 1, 2 and many cells per axis,
the periodic stencil on either side of wrapping onto itself, planar and linear catalogues, cell keys above 32 bits and
the per-axis caps, cells of exactly 127 .. 257 rows around the kernels' chunk of 128 primaries, and float32 catalogues
far from the origin.  FOF labels and npairs match exactly; the pair sums to rtol 1e-12 and zeta to 1e-9 B.

Every test also checks that its case occurred on the grid the run built (cells per axis, key bits, rows per cell, a row
on L_f4), and that every row lies inside its cell: FOF links all rows of one cell without testing their distance, and
the pair kernels allow a row `tol` outside its cell."""
import math

import numpy as np
import pytest
import torch

from oracle import fof_oracle as fo  # noqa: E402
from oracle import paircount_oracle as po  # noqa: E402
from oracle import threeptcf_oracle as to  # noqa: E402

pytestmark = pytest.mark.gpu

_COMM = []
L_UP = 100.0014       # float32(L_UP) = L_UP + 3.8e-6
L_DOWN = 100.0013     # float32(L_DOWN) = L_DOWN - 3.0e-6


def _comm():
    from nbodykit_b200.comm import SelfComm
    if not _COMM:
        _COMM.append(SelfComm())
    return _COMM[0]


def _cat(pos, w=None, box=None):
    from nbodykit_b200.lab import ArrayCatalog
    data = {"Position": torch.as_tensor(np.ascontiguousarray(pos)).cuda()}
    if w is not None:
        data["Weight"] = torch.as_tensor(np.ascontiguousarray(w)).cuda()
    kw = dict(BoxSize=np.asarray(box, "f8")) if box is not None else {}
    return ArrayCatalog(data, comm=_comm(), **kw)


def _f4(L):
    return float(np.float32(L))


# ---- what the runs built -----------------------------------------------------------------------------------------------
@pytest.fixture
def grids(monkeypatch, cuda):
    """records the cell grids of every run: FOF's (box, origin, cells per axis, key of every row) and every pair grid's
    (box, origin, cells per axis, tol, sorted positions, occupied keys, rows per cell)"""
    from nbodykit_b200.algorithms import fof, paircount, threeptcf
    rec = dict(fof=[], pair=[])
    local_fof, sort_rows = fof._local_fof, fof._sort_rows

    def rec_local_fof(pos, gid, gid_base, periodic, box, origin, b, want_minid):
        rec["fof"].append(dict(pos=pos.cpu().numpy(), periodic=bool(periodic), box=np.array(box, "f8"),
                               origin=np.array(origin, "f8"), ncell=fof._cells(box, b)))
        return local_fof(pos, gid, gid_base, periodic, box, origin, b, want_minid)

    def rec_sort_rows(keys, key_bytes, end_bit):
        if key_bytes == 8 and rec["fof"] and "keys" not in rec["fof"][-1]:
            rec["fof"][-1]["keys"] = keys.cpu().numpy().copy()
        return sort_rows(keys, key_bytes, end_bit)

    class Cells(paircount._Cells):
        def __init__(self, pos, w, periodic, box, origin, ncell):
            super().__init__(pos, w, periodic, box, origin, ncell)
            box, origin = np.array(box, "f8"), np.array(origin, "f8")
            rec["pair"].append(dict(pos=self.pos.cpu().numpy(), periodic=bool(periodic), box=box, origin=origin,
                                    ncell=[int(v) for v in ncell], tol=4e-7 * (box + np.abs(origin)),
                                    keys=self.cell_key.cpu().numpy(),
                                    sizes=np.diff(self.cell_start.to(torch.int64).cpu().numpy())))

    monkeypatch.setattr(fof, "_local_fof", rec_local_fof)
    monkeypatch.setattr(fof, "_sort_rows", rec_sort_rows)
    monkeypatch.setattr(paircount, "_Cells", Cells)
    monkeypatch.setattr(threeptcf, "_Cells", Cells)
    return rec


def _outside(pos, keys, ncell, box, origin, periodic):
    """per row and axis, how far the row lies outside the cell of its key (minimum image when periodic)"""
    nc = np.asarray(ncell, np.int64)
    keys = np.asarray(keys, np.int64)
    idx = np.stack([keys // (nc[1] * nc[2]), (keys // nc[2]) % nc[1], keys % nc[2]], 1)
    cs = box / nc
    d = np.asarray(pos, "f8") - (origin + (idx + 0.5) * cs)
    if periodic:
        d = d - box * np.round(d / box)
    return np.maximum(np.abs(d) - 0.5 * cs, 0.)


def _fof_grid(g):
    """FOF's grid of one run, after checking that every row lies inside its cell to double rounding"""
    pos = fo.wrapped(g["pos"], g["box"]) if g["periodic"] else g["pos"]
    out = _outside(pos, g["keys"], g["ncell"], g["box"], g["origin"], g["periodic"])
    assert out.max() <= 1e-12 * float(np.max(g["box"] + np.abs(g["origin"]))), out.max()
    return g


def _pair_grids(rec):
    """the pair grids of one run, after checking that every row lies within tol of its cell"""
    for g in rec["pair"]:
        keys = np.repeat(g["keys"], g["sizes"])
        out = _outside(g["pos"], keys, g["ncell"], g["box"], g["origin"], g["periodic"])
        assert (out <= g["tol"]).all(), out.max(0)
    return rec["pair"]


def _key_bits(keys):
    return int(np.max(keys)).bit_length()


def _fof(pos, b, nmin=0, box=None, periodic=True):
    from nbodykit_b200.lab import FOF
    f = FOF(_cat(pos, box=box if periodic else None), linking_length=b, nmin=nmin, absolute=True, periodic=periodic)
    want = fo.fof_labels(pos, b, nmin, box if periodic else None)
    np.testing.assert_array_equal(f.labels, want)
    return f, want


def _pairs(mode, pos, edges, box, periodic=True, los=2, brute=False, w=None, **kw):
    from nbodykit_b200.lab import SimulationBoxPairCount
    r = SimulationBoxPairCount(mode, _cat(pos, w, box), edges, BoxSize=box, periodic=periodic, los=los, **kw)
    oracle = po.brute_force if brute else po.count
    want = oracle(pos, mode, edges, box if periodic else None, w1=w, los=los, **kw)
    p = r.pairs
    np.testing.assert_array_equal(p["npairs"], want["npairs"])
    np.testing.assert_allclose(p["wnpairs"], want["wnpairs"], rtol=1e-12, atol=0)
    n = want["npairs"]
    np.testing.assert_allclose(p[p.dims[0]], np.where(n > 0, want["sepsum"] / np.maximum(n, 1), 0.), rtol=1e-12, atol=0)
    assert want["npairs"].sum() > 0
    return r, want


def _3pcf(pos, edges, poles, box, periodic=True, brute=False, w=None):
    from nbodykit_b200.lab import SimulationBox3PCF
    r = SimulationBox3PCF(_cat(pos, w, box), poles, edges, BoxSize=box, periodic=periodic)
    oracle = to.brute_force if brute else to.compute
    want = oracle(pos, edges, poles, box=box if periodic else None, w=w)
    np.testing.assert_array_equal(r.npairs, want["npairs"])
    z = np.stack([r.poles["corr_%d" % ell] for ell in poles])
    err = np.abs(z - want["zeta"])
    assert (err <= 1e-9 * want["bound"]).all(), float(np.max(err / np.maximum(want["bound"], 1e-300)))
    assert want["npairs"].sum() > 0
    return r, want


def _edge_rows(rng, L, n):
    """float32 rows with one to three coordinates at 0, at tiny negatives that wrap onto L_f4, at L_f4 or one ulp below
    it, the others uniform"""
    Lf = np.float32(L)
    vals = np.array([0., -1e-9, -3e-8, -np.float32(1e-30), Lf, np.nextafter(Lf, np.float32(0))], "f4")
    pos = (rng.uniform(size=(n, 3)) * L).astype("f4")
    for i in range(n):
        axes = rng.choice(3, size=rng.randint(1, 4), replace=False)
        pos[i, axes] = rng.choice(vals, size=len(axes))
    return pos


def _assert_wraps_onto_L_f4(pos, L):
    """some row's float32 coordinate is below 0 and wraps onto L_f4 under `pos % L`"""
    Lf = np.float32(L)
    w = np.mod(pos, Lf)
    assert ((pos < 0) & (w == Lf)).any()


# ---- 1. box sides float32 cannot hold ----------------------------------------------------------------------------------
def test_fof_f4_row_wrapped_onto_L_f4_is_not_linked_inside_its_cell(grids):
    """regression: a float32 row at -1e-9 wraps onto L_f4 = L + 3.8e-6.  Clamped into the last cell, it shared cell
    (2, 2, 2) with a row 7e-8 b^2 beyond the linking length and was linked to it"""
    L = L_UP
    assert _f4(L) - L > 3e-6
    b = L * math.sqrt(3) * (1 + 2e-9) / 3
    pos = np.array([[-1e-9] * 3, [66.6676025390625] * 3], "f4")
    _assert_wraps_onto_L_f4(pos, L)
    f, want = _fof(pos, b, 0, [L] * 3)
    np.testing.assert_array_equal(want, [1, 2])
    np.testing.assert_array_equal(f.labels, [1, 2])
    g = _fof_grid(grids["fof"][0])
    assert g["ncell"] == [3, 3, 3]
    # the second row is in the last cell on every axis
    assert g["keys"][1] == 26


@pytest.mark.parametrize("L", [L_UP, L_DOWN], ids=["Lf4_above_L", "Lf4_below_L"])
def test_fof_box_side_not_exact_in_f4(grids, L):
    """2000 float32 rows plus 200 at 0, at tiny negatives, at L_f4 and one ulp below it, with b at the smallest cell
    margin (40 cells of side b / sqrt(3) / (1 + 1e-9))"""
    rng = np.random.RandomState(11)
    pos = np.concatenate([(rng.uniform(size=(2000, 3)) * L).astype("f4"), _edge_rows(rng, L, 200)])
    _assert_wraps_onto_L_f4(pos, L)
    assert (pos == np.nextafter(np.float32(L), np.float32(0))).any()
    b = L * math.sqrt(3) * (1 + 2e-9) / 40
    f, want = _fof(pos, b, 1, [L] * 3)
    g = _fof_grid(grids["fof"][0])
    assert g["ncell"] == [40, 40, 40]
    assert want.max() > 10


@pytest.mark.parametrize("mode", ["1d", "2d", "projected"])
@pytest.mark.parametrize("L", [L_UP, L_DOWN], ids=["Lf4_above_L", "Lf4_below_L"])
def test_pairs_box_side_not_exact_in_f4(grids, mode, L):
    rng = np.random.RandomState(12)
    pos = np.concatenate([(rng.uniform(size=(3000, 3)) * L).astype("f4"), _edge_rows(rng, L, 300)])
    _assert_wraps_onto_L_f4(pos, L)
    kw = dict(Nmu=5) if mode == "2d" else (dict(pimax=6.) if mode == "projected" else {})
    _pairs(mode, pos, np.linspace(0.9, 9.7, 7), [L] * 3, los=[2, 0, 1][len(mode) % 3], **kw)
    for g in _pair_grids(grids):
        # the wrapped row sits on L_f4 in the sorted positions the kernel reads
        assert (g["pos"] == _f4(L)).any()


def test_3pcf_noncubic_box_sides_not_exact_in_f4(grids):
    """a periodic box with one side above its float32 value, one below and one exact"""
    box = np.array([L_UP, L_DOWN, 60.])
    rng = np.random.RandomState(13)
    pos = np.concatenate([(rng.uniform(size=(2500, 3)) * box).astype("f4"), _edge_rows(rng, L_UP, 150) * [1, 1, 0.5]])
    pos = pos.astype("f4")
    _assert_wraps_onto_L_f4(pos[:, :1], L_UP)
    _3pcf(pos, np.linspace(0., 9., 5), [0, 1, 2, 5], box)
    (g,) = _pair_grids(grids)
    assert (g["pos"][:, 0] == _f4(L_UP)).any() and (g["pos"][:, 1] == _f4(L_DOWN)).any()


# ---- 2. cell counts at their limits ------------------------------------------------------------------------------------
@pytest.mark.parametrize("side", ["b_below", "b_above"])
def test_fof_cell_count_at_ceil_boundary(grids, side):
    """b a relative 1e-11 either side of the b that gives exactly 13 cells: 14 cells below it, 13 above it, and pairs
    at opposite corners of one cell (sqrt(3) of its side apart) linked"""
    L, n = 20., 13
    b0 = L * math.sqrt(3) * (1 + 1e-9) / n
    b = b0 * (1 - 1e-11 if side == "b_below" else 1 + 1e-11)
    rng = np.random.RandomState(14)
    cs = L / n
    k = rng.randint(0, n, size=(40, 3))
    corners = np.concatenate([k * cs, (k + 1) * cs])             # opposite corners of 40 cells
    pos = np.concatenate([rng.uniform(size=(250, 3)) * L, corners])
    f, want = _fof(pos, b, 0, [L] * 3)
    assert (want[250:290] == want[290:]).all()
    assert 5 < want.max() < len(pos)
    g = _fof_grid(grids["fof"][0])
    assert g["ncell"] == [n + 1 if side == "b_below" else n] * 3


@pytest.mark.parametrize("box", [[0.18, 0.38, 30.], [30., 0.18, 0.38], [0.38, 30., 0.18]], ids=["xyz", "yzx", "zxy"])
def test_fof_noncubic_one_two_many_cells(grids, box):
    """a periodic box with 1, 2 and 149 cells on different axes: the stencil visits the first two whole and wraps the
    third"""
    b = 0.35
    rng = np.random.RandomState(15)
    pos = rng.uniform(size=(70, 3)) * box
    pos = np.concatenate([pos, [[0., 0., 0.], np.asarray(box) - 1e-9, [-1e-12] * 3]])
    f, want = _fof(pos, b, 0, box)
    g = _fof_grid(grids["fof"][0])
    order = np.argsort(box)
    assert [g["ncell"][i] for i in order] == [1, 2, 149]
    reach = [math.floor(b / (s / c) * (1 + 1e-12)) + 1 for s, c in zip(box, g["ncell"])]
    full = [2 * r + 1 >= c for r, c in zip(reach, g["ncell"])]
    assert [full[i] for i in order] == [True, True, False]
    assert 1 < want.max() < len(pos)


def _plane(rng, n):
    p = rng.uniform(size=(n, 3)) * 30.
    p[:, 2] = 3.7
    return p


def _line(rng, n):
    p = np.zeros((n, 3)) + [1.5, -2.25, 8.]
    p[:, 0] = rng.uniform(size=n) * 200.
    return p


@pytest.mark.parametrize("shape", ["plane", "line"])
def test_fof_nonperiodic_plane_and_line(grids, shape):
    """all z equal (the grid takes a side of 1 there), or all rows on a line along x"""
    rng = np.random.RandomState(16)
    pos = _plane(rng, 1500) if shape == "plane" else _line(rng, 600)
    f, want = _fof(pos, 0.5, 0, periodic=False)
    g = _fof_grid(grids["fof"][0])
    flat = [2] if shape == "plane" else [1, 2]
    for d in flat:
        assert g["box"][d] == 1. and g["ncell"][d] == 4
    assert 1 < want.max() < len(pos)


@pytest.mark.parametrize("ncell", [3, 4, 5, 6])
def test_pairs_periodic_cells_around_self_wrap(grids, ncell):
    """3 to 6 cells per axis: the stencil of 2 reach + 1 cells wraps onto itself up to 5 cells and not at 6"""
    L = 30.
    smax = L / 2 if ncell == 3 else 2 * L / (ncell + 0.5) / 1.0001
    rng = np.random.RandomState(17 + ncell)
    pos = np.concatenate([rng.uniform(size=(1200, 3)) * L, [[0., 0., 0.], [L, L, L], [-1e-9, L / 2, L - 1e-9]]])
    mode = "1d" if ncell % 2 else "2d"
    _pairs(mode, pos, np.linspace(0.5, smax, 6), [L] * 3, brute=True, **(dict(Nmu=4) if mode == "2d" else {}))
    for g in _pair_grids(grids):
        assert g["ncell"] == [ncell] * 3
        cs = L / ncell
        reach = math.floor((smax + 2 * g["tol"][0]) / cs * (1 + 1e-12)) + 1
        assert (2 * reach + 1 >= ncell) == (ncell <= 5)


@pytest.mark.parametrize("ncell", [1, 2])
def test_pairs_nonperiodic_one_and_two_cells(grids, ncell):
    L = 30.
    smax = 2 * L / (ncell + 0.5) / 1.0001
    rng = np.random.RandomState(21 + ncell)
    pos = np.concatenate([rng.uniform(size=(800, 3)) * L, [[0., 0., 0.], [L, L, L]]])
    mode = "1d" if ncell == 1 else "2d"
    _pairs(mode, pos, np.linspace(0.5, smax, 5), [L] * 3, periodic=False, brute=True,
           **(dict(Nmu=3) if mode == "2d" else {}))
    for g in _pair_grids(grids):
        assert g["ncell"] == [ncell] * 3


@pytest.mark.parametrize("shape", ["plane", "line"])
def test_pairs_nonperiodic_plane_and_line(grids, shape):
    rng = np.random.RandomState(23)
    pos = _plane(rng, 1500) if shape == "plane" else _line(rng, 800)
    mode, kw = ("2d", dict(Nmu=4)) if shape == "plane" else ("1d", {})
    _pairs(mode, pos, np.linspace(0.3, 3., 6), [30.] * 3, periodic=False, **kw)
    for g in _pair_grids(grids):
        for d in ([2] if shape == "plane" else [1, 2]):
            assert g["box"][d] == 1. and g["ncell"][d] == 1
        assert max(g["ncell"]) > 10


def test_3pcf_noncubic_cells_around_self_wrap(grids):
    """3, 4 and 7 cells on the three axes: the first two visited whole, the third wrapped"""
    box = np.array([30., 36., 60.])
    rng = np.random.RandomState(24)
    pos = np.concatenate([rng.uniform(size=(500, 3)) * box, [[0., 0., 0.], box, [-1e-9, 18., 60. - 1e-9]]])
    _3pcf(pos, np.linspace(0., 15., 4), [0, 2, 3], box, brute=True)
    (g,) = _pair_grids(grids)
    assert g["ncell"] == [3, 4, 7]


def test_3pcf_nonperiodic_plane(grids):
    rng = np.random.RandomState(25)
    _3pcf(_plane(rng, 700), np.linspace(0., 3., 4), [0, 1, 2, 4], [30.] * 3, periodic=False, brute=True)
    (g,) = _pair_grids(grids)
    assert g["box"][2] == 1.


# ---- 3. keys above 32 bits ---------------------------------------------------------------------------------------------
def _clumps(rng, far, n, scale, dtype="f8"):
    """two gaussian clumps of n rows, the second `far` away on every axis"""
    a = rng.normal(scale=scale, size=(n, 3))
    b = rng.normal(scale=scale, size=(n, 3)) + far
    return np.concatenate([a, b]).astype(dtype)


def test_fof_far_clumps_keys_above_32_bits(grids):
    """two clumps 1e6 b apart on every axis: 1.73e6 cells per axis (the cap is 2^21), keys of 62 bits"""
    b = 0.3
    rng = np.random.RandomState(31)
    pos = _clumps(rng, 1e6 * b, 400, 1.)
    f, want = _fof(pos, b, 0, periodic=False)
    g = _fof_grid(grids["fof"][0])
    assert all((1 << 20) < c <= (1 << 21) for c in g["ncell"])
    assert _key_bits(g["keys"]) >= 60
    assert 2 < want.max() < len(pos)


def test_fof_sparse_periodic_tiny_b_keys_above_32_bits(grids):
    """b = 1e-4 in L = 100: 1.73e6 cells per axis, keys of about 2^62; pairs and chains inside and across the faces"""
    L, b = 100., 1e-4
    rng = np.random.RandomState(32)
    base = rng.uniform(size=(1500, 3)) * L
    u = rng.normal(size=(1500, 3))
    u /= np.linalg.norm(u, axis=1)[:, None]
    step = b * rng.uniform(0.3, 0.95, size=(1500, 1)) * u
    faces = np.array([[1e-5, 50., 50.], [L - 4e-5, 50., 50.], [L - 1e-5, L - 1e-5, L - 1e-5], [2e-5, 3e-5, 1e-5]])
    pos = np.concatenate([base, base[:700] + step[:700], base[:300] + 2 * step[:300], faces]) % L
    f, want = _fof(pos, b, 0, [L] * 3)
    g = _fof_grid(grids["fof"][0])
    assert all((1 << 20) < c <= (1 << 21) for c in g["ncell"])
    assert _key_bits(g["keys"]) >= 60
    assert want[-4] == want[-3] and want[-2] == want[-1]
    assert np.bincount(want).max() == 3


def _extent_for(cells, b):
    """a non-periodic x extent that gives exactly `cells` FOF cells per axis"""
    return (cells - 0.5) * b / (math.sqrt(3) * (1 + 1e-9))


def test_fof_cells_per_axis_cap(grids):
    """2^21 cells along x are accepted (keys up to 2^21 - 1 times the other axes), 2^21 + 1 raise ValueError"""
    b = 1.
    e = _extent_for(1 << 21, b)
    pos = np.array([[0., 0., 0.], [0.2, 0., 0.], [e, 0., 0.], [e - 0.5, 0., 0.]])
    f, want = _fof(pos, b, 0, periodic=False)
    np.testing.assert_array_equal(want, [1, 1, 2, 2])
    g = _fof_grid(grids["fof"][0])
    assert g["ncell"] == [1 << 21, 2, 2]
    assert int(g["keys"].max()) == ((1 << 21) - 1) * 4
    from nbodykit_b200.lab import FOF
    pos[2:, 0] = _extent_for((1 << 21) + 1, b) - np.array([0., 0.5])
    with pytest.raises(ValueError, match="63-bit"):
        FOF(_cat(pos), linking_length=b, nmin=0, absolute=True, periodic=False)


@pytest.mark.parametrize("far", [1e5, 1e6])
def test_pairs_far_clumps_keys_above_32_bits(grids, far):
    """two clumps `far` s_max apart on every axis: 2e5 cells per axis, or the cap of 2^20"""
    smax = 2.
    rng = np.random.RandomState(33)
    pos = _clumps(rng, far * smax, 300, 0.7)
    _pairs("1d", pos, np.linspace(0.1, smax, 5), [1.] * 3, periodic=False)
    _pairs("projected", pos, np.linspace(0.1, 1.4, 5), [1.] * 3, periodic=False, pimax=1.4)
    for g in _pair_grids(grids):
        assert _key_bits(g["keys"]) > 32
        assert g["ncell"] == [1 << 20] * 3 if far == 1e6 else all(1e5 < c < (1 << 20) for c in g["ncell"])


@pytest.mark.parametrize("far", [1e5, 1e6])
def test_3pcf_far_clumps_keys_above_32_bits(grids, far):
    rmax = 2.
    rng = np.random.RandomState(34)
    pos = _clumps(rng, far * rmax, 250, 0.7)
    _3pcf(pos, np.linspace(0., rmax, 5), [0, 1, 3], [1.] * 3, periodic=False)
    (g,) = _pair_grids(grids)
    assert _key_bits(g["keys"]) > 32
    assert g["ncell"] == [1 << 20] * 3 if far == 1e6 else all(1e5 < c < (1 << 20) for c in g["ncell"])


# ---- 4. chunk and tile boundaries --------------------------------------------------------------------------------------
_CELL_ROWS = [127, 128, 129, 256, 257]


def _chunk_catalogue(seed, L, nc):
    """cells of exactly 127, 128, 129, 256 and 257 rows (a tight clump in each, half of its rows duplicates) and a
    background in the other cells, on the periodic grid of nc cells per axis"""
    rng = np.random.RandomState(seed)
    cs = L / nc
    cells = rng.choice(nc ** 3, size=len(_CELL_ROWS), replace=False)
    parts = []
    for c, n in zip(cells, _CELL_ROWS):
        centre = (np.array(np.unravel_index(c, (nc,) * 3)) + 0.5) * cs
        u = centre + np.clip(rng.normal(scale=0.1 * cs, size=((n + 1) // 2, 3)), -0.4 * cs, 0.4 * cs)
        parts.append(np.concatenate([u, u[:n // 2]]))
    bg = rng.uniform(size=(600, 3)) * L
    key = np.ravel_multi_index(tuple(np.minimum((bg / cs).astype(int), nc - 1).T), (nc,) * 3)
    parts.append(bg[~np.isin(key, cells)])
    return np.concatenate(parts)


def _assert_cell_rows(g, chunk):
    """the grid holds cells of exactly 127 .. 257 rows, so some cells end in a partial chunk of primaries"""
    for n in _CELL_ROWS:
        assert n in g["sizes"]
    assert chunk == 128
    assert set((g["sizes"] % chunk).tolist()) >= {1, 127}


@pytest.mark.parametrize("mode", ["1d", "2d"])
def test_pairs_cells_at_chunk_boundaries(grids, mode):
    from nbodykit_b200._lib import lib
    L, smax = 40., 4.
    nc = math.floor(2 * L / (smax * 1.0001))
    pos = _chunk_catalogue(41, L, nc)
    w = np.random.RandomState(42).uniform(0.5, 2., len(pos))
    _pairs(mode, pos, np.linspace(0.05, smax, 6), [L] * 3, w=w, **(dict(Nmu=5) if mode == "2d" else {}))
    for g in _pair_grids(grids):
        assert g["ncell"] == [nc] * 3
        _assert_cell_rows(g, int(lib().nbk_paircount_chunk_rows()))


def test_3pcf_cells_at_chunk_boundaries(grids):
    """chunks of 127 and 1 primaries: row counts that are not a multiple of the warps per CTA"""
    from nbodykit_b200._lib import lib
    L, rmax = 40., 4.
    nc = math.floor(2 * L / (rmax * 1.0001))
    pos = _chunk_catalogue(43, L, nc)
    w = np.random.RandomState(44).uniform(-1., 2., len(pos))
    _3pcf(pos, np.linspace(0., rmax, 5), [0, 1, 2, 7], [L] * 3, w=w)
    (g,) = _pair_grids(grids)
    assert g["ncell"] == [nc] * 3
    _assert_cell_rows(g, int(lib().nbk_threeptcf_chunk_rows()))


# ---- 5. far-off origins ------------------------------------------------------------------------------------------------
_OFFSET = np.array([1e5, -4e5, 1e6])


def _far_f4(seed, n):
    """a clustered float32 catalogue offset by 1e5 .. 1e6, where the float32 spacing is 1/128 .. 1/16"""
    rng = np.random.RandomState(seed)
    p = np.concatenate([rng.uniform(size=(n // 2, 3)) * 30., rng.normal(scale=1.5, size=(n // 2, 3)) + 15.])
    return (p + _OFFSET).astype("f4")


def test_fof_far_off_origin_f4(grids):
    pos = _far_f4(51, 3000)
    f, want = _fof(pos, 0.61, 1, periodic=False)
    g = _fof_grid(grids["fof"][0])
    assert np.all(np.abs(g["origin"]) > 9e4)
    assert 5 < want.max() < len(pos)


@pytest.mark.parametrize("mode", ["1d", "2d", "projected"])
def test_pairs_far_off_origin_f4(grids, mode):
    pos = _far_f4(52, 2500)
    kw = dict(Nmu=4) if mode == "2d" else (dict(pimax=2.) if mode == "projected" else {})
    _pairs(mode, pos, np.linspace(0.37, 2.9, 6), [1.] * 3, periodic=False, **kw)
    for g in _pair_grids(grids):
        assert np.all(np.abs(g["origin"]) > 9e4)


def test_3pcf_far_off_origin_f4(grids):
    pos = _far_f4(53, 1500)
    _3pcf(pos, np.linspace(0., 2.5, 5), [0, 2, 4], [1.] * 3, periodic=False)
    (g,) = _pair_grids(grids)
    assert np.all(np.abs(g["origin"]) > 9e4)
