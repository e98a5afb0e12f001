"""The cell grids and neighbour walks of the survey pair counts, CylindricalGroups, KDDensity and FiberCollisions at their
edges, against the float64 CPU restatements in oracle/: every histogram size on either side of the shared-memory limit
of csrc/paircount.cu, cells of exactly 127 .. 257 rows around the chunk of 128 primaries of the pair and CGM kernels,
pi exactly at pimax, pairs found only through the sphere prune of survey 'projected', thin shells far from the observer,
angles up to 180 degrees; periodic box sides float32 cannot hold, non-cubic boxes, sparse catalogues whose widened CGM
grid has 1, 2 or 3 cells per axis, z reaches that wrap at both faces, zero-radius cylinders; KDDensity cell counts at
their row boundaries, neighbours found only in the last ring of an even or odd grid, rows on cell faces and rows whose
unit coordinate rounds to 1.0; FiberCollisions groups at and around the sizes where the greedy changes path, ties of the
nearest uncollided member, collision radii that leave 1, 2 or 3 cells per axis and pairs a relative 1e-12 from the
radius; and rows on the x-slab boundaries of two and three ranks.

Tolerances are those of each algorithm's own tests: CGM labels, KDDensity distances and FiberCollisions outputs bit for
bit, density to 1e-15, npairs exactly and the pair sums to rtol 1e-12.  Every test also checks that its case occurred on
the grid the run built (cells per axis, rows per cell, the histogram side, group sizes, a row on L_f4).

Two limits these tests cannot reach: CGM cell keys above 32 bits cannot occur, because its sparse-catalogue widening keeps
about n / 16 cells; and KDDensity's cap of 1024 cells per axis needs 4 * 1024^3 rows, above the 2^31 - 1 rows per rank."""
import math
import warnings

import numpy as np
import pytest
import torch

from oracle import cgm_oracle as co
from oracle import fibercollisions_oracle as fo
from oracle import kddensity_oracle as ko
from oracle import paircount_oracle as po
from oracle import survey_paircount_oracle as so
from test_gpu_cell_grid_edges import L_DOWN, L_UP, _assert_wraps_onto_L_f4, _edge_rows, _f4, _outside

pytestmark = pytest.mark.gpu

_COMM = []
# rows per cell around the chunk of 128 primaries of csrc/paircount.cu and csrc/cgm.cu
_CELL_ROWS = [127, 128, 129, 255, 256, 257]


def _comm():
    from nbodykit_b200.comm import SelfComm
    if not _COMM:
        _COMM.append(SelfComm())
    return _COMM[0]


def _lib():
    from nbodykit_b200._lib import lib
    return lib()


# ---- what the runs built -----------------------------------------------------------------------------------------------
@pytest.fixture
def grids(monkeypatch, cuda):
    """records every cell grid the pair counts, CylindricalGroups and KDDensity build: box, origin, cells per axis,
    tol, sorted positions, occupied keys and rows per cell"""
    from nbodykit_b200.algorithms import cgm, kdtree, paircount
    rec = []

    class Cells(paircount._Cells):
        def __init__(self, pos, w, periodic, box, origin, ncell):
            super().__init__(pos, w, periodic, box, origin, ncell)
            box, origin = np.array(box, "f8"), np.array(origin, "f8")
            rec.append(dict(pos=self.pos.cpu().numpy(), periodic=bool(periodic), box=box, origin=origin,
                            ncell=[int(v) for v in ncell], tol=4e-7 * (box + np.abs(origin)),
                            keys=self.cell_key.cpu().numpy(),
                            sizes=np.diff(self.cell_start.to(torch.int64).cpu().numpy())))

    for m in (cgm, kdtree, paircount):
        monkeypatch.setattr(m, "_Cells", Cells)
    return rec


def _checked(rec):
    """the recorded grids, after checking that every row lies within tol of its cell"""
    assert rec
    for g in rec:
        keys = np.repeat(g["keys"], g["sizes"])
        out = _outside(g["pos"], keys, g["ncell"], g["box"], g["origin"], g["periodic"])
        assert (out <= g["tol"]).all(), out.max(0)
    return rec


def _assert_cell_rows(g, chunk):
    """the grid holds cells of exactly 127 .. 257 rows, so some cells end in a partial chunk of 1 or 127 primaries"""
    assert chunk == 128
    for n in _CELL_ROWS:
        assert n in g["sizes"], n
    assert set((g["sizes"] % chunk).tolist()) >= {1, 127}


# ---- survey pair counts --------------------------------------------------------------------------------------------------
def _sky_cat(ra, dec, z=None, w=None, dtype="f8", comm=None):
    from nbodykit_b200.lab import ArrayCatalog
    data = {"RA": torch.as_tensor(np.ascontiguousarray(ra, dtype)).cuda(),
            "DEC": torch.as_tensor(np.ascontiguousarray(dec, dtype)).cuda()}
    if z is not None:
        data["Redshift"] = torch.as_tensor(np.ascontiguousarray(z, dtype)).cuda()
    if w is not None:
        data["Weight"] = torch.as_tensor(np.ascontiguousarray(w, "f8")).cuda()
    return ArrayCatalog(data, comm=comm or _comm())


def _sky_rows(mode, ra, dec, z, dtype="f8"):
    """the float64 rows the survey count bins: SkyToCartesian (SkyToUnitSphere for 'angular') of the columns as stored"""
    from nbodykit_b200 import transform as T
    from nbodykit_b200.cosmology import Planck15
    t = [torch.as_tensor(np.ascontiguousarray(a, dtype)).cuda() for a in ((ra, dec) if mode == "angular" else (ra, dec, z))]
    p = T.SkyToUnitSphere(t[0], t[1]) if mode == "angular" else T.SkyToCartesian(t[0], t[1], t[2], Planck15)
    return p.cpu().numpy()


def _to_sky(rows, mode):
    """(ra, dec, z) of Cartesian rows ('angular': (ra, dec, None) of unit vectors)"""
    if mode == "angular":
        ra = np.rad2deg(np.arctan2(rows[:, 1], rows[:, 0])) % 360.
        return ra, np.rad2deg(np.arcsin(np.clip(rows[:, 2], -1., 1.))), None
    from nbodykit_b200 import transform as T
    from nbodykit_b200.cosmology import Planck15
    ra, dec, z = T.CartesianToSky(torch.from_numpy(np.ascontiguousarray(rows, "f8")).cuda(), Planck15)
    return ra.cpu().numpy(), dec.cpu().numpy(), z.cpu().numpy()


def _compare(p, want):
    np.testing.assert_array_equal(p["npairs"], want["npairs"])
    np.testing.assert_allclose(p["wnpairs"], want["wnpairs"], rtol=1e-12, atol=0)
    n = want["npairs"]
    np.testing.assert_allclose(p[p.dims[0]], np.where(n > 0, want["sepsum"] / np.maximum(n, 1), 0.), rtol=1e-12, atol=0)
    assert n.sum() > 0


def _survey(mode, s1, edges, s2=None, w1=None, w2=None, dtype="f8", brute=False, **kw):
    """SurveyDataPairCount of sky columns s1 (and s2) against the oracle on the rows the count bins"""
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200.lab import SurveyDataPairCount
    z1 = None if mode == "angular" else s1[2]
    second = None if s2 is None else _sky_cat(s2[0], s2[1], None if mode == "angular" else s2[2], w2, dtype)
    r = SurveyDataPairCount(mode, _sky_cat(s1[0], s1[1], z1, w1, dtype), edges, cosmo=Planck15, second=second, **kw)
    oracle = so.brute_force if brute else so.count
    want = oracle(_sky_rows(mode, *s1, dtype=dtype), mode, edges,
                  pos2=None if s2 is None else _sky_rows(mode, *s2, dtype=dtype), w1=w1, w2=w2, **kw)
    _compare(r.pairs, want)
    return r, want


def _box(mode, pos, edges, L, pos2=None, w1=None, w2=None, **kw):
    from nbodykit_b200.lab import ArrayCatalog, SimulationBoxPairCount

    def cat(p, w):
        return ArrayCatalog({"Position": torch.from_numpy(p).cuda(), "Weight": torch.from_numpy(w).cuda()},
                            comm=_comm(), BoxSize=[L] * 3)
    r = SimulationBoxPairCount(mode, cat(pos, w1), edges, BoxSize=L, periodic=True,
                               second=None if pos2 is None else cat(pos2, w2), **kw)
    want = po.count(pos, mode, edges, [L] * 3, pos2=pos2, w1=w1, w2=w2, **kw)
    _compare(r.pairs, want)
    return r, want


# histogram shapes (first, second dimension) at, just above and well above the shared-memory limit of 1024 bins
_SHAPES = {"at": ((1024, 1), (32, 32)), "above": ((1025, 1), (25, 41)), "far": ((4000, 1), (64, 64))}


def _hist_kw(mode, side, emax):
    (nb1, _), (nb, n2) = _SHAPES[side]
    if mode in ("1d", "angular"):
        return np.linspace(emax / 80., emax, nb1 + 1), {}
    e = np.linspace(emax / 80., emax, nb + 1)
    return e, (dict(Nmu=n2) if mode == "2d" else dict(pimax=float(n2)))


def _assert_side(r, side):
    smem = int(_lib().nbk_paircount_smem_bins())
    assert smem == 1024
    nbins = int(np.prod(r.pairs.shape))
    assert nbins == {"at": smem, "above": smem + 1}.get(side, nbins)
    assert (nbins <= smem) == (side == "at")
    assert side != "far" or nbins > 3 * smem


@pytest.mark.parametrize("side", ["at", "above", "far"])
@pytest.mark.parametrize("mode", ["1d", "2d", "projected", "angular"])
def test_survey_histogram_either_side_of_shared_memory(grids, mode, side):
    """auto and cross counts, weighted, with nbins = 1024 (shared-memory histogram), 1025 and >= 4000 (global atomics)"""
    rng = np.random.RandomState(300 + len(mode))
    s1 = so.sky_catalogue(301, 1500, ra=(20., 40.), dec=(10., 25.), z=(0.05, 0.01))
    s2 = so.sky_catalogue(302, 1000, ra=(20., 40.), dec=(10., 25.), z=(0.05, 0.01))
    w1, w2 = rng.uniform(0.5, 2., 1500), rng.uniform(0.5, 2., 1000)
    edges, kw = _hist_kw(mode, side, 12. if mode == "angular" else 40.)
    r, want = _survey(mode, s1, edges, w1=w1, **kw)
    _assert_side(r, side)
    r, want = _survey(mode, s1, edges, s2=s2, w1=w1, w2=w2, **kw)
    _assert_side(r, side)
    # the counts reach far into the histogram, beyond the first 1024 bins when there are more
    assert np.nonzero(want["npairs"].reshape(-1))[0].max() > min(1000, want["npairs"].size // 2)
    _checked(grids)


@pytest.mark.parametrize("side", ["at", "above", "far"])
@pytest.mark.parametrize("mode", ["1d", "projected"])
def test_box_histogram_either_side_of_shared_memory(grids, mode, side):
    rng = np.random.RandomState(310 + len(mode))
    L = 150.
    pos1, pos2 = rng.uniform(size=(2000, 3)) * L, rng.uniform(size=(1200, 3)) * L
    w1, w2 = rng.uniform(0.5, 2., 2000), rng.uniform(0.5, 2., 1200)
    edges, kw = _hist_kw(mode, side, 20.)
    r, want = _box(mode, pos1, edges, L, w1=w1, **kw)
    _assert_side(r, side)
    r, want = _box(mode, pos1, edges, L, pos2=pos2, w1=w1, w2=w2, **kw)
    _assert_side(r, side)
    assert np.nonzero(want["npairs"].reshape(-1))[0].max() > min(1000, want["npairs"].size // 2)
    _checked(grids)


def _survey_grid(rows, smax):
    """(lo, cs, ncell) of the non-periodic grid count_pairs builds over `rows`"""
    lo, hi = rows.min(0), rows.max(0)
    gbox = np.where(hi > lo, hi - lo, 1.0)
    nc = np.array([int(min(max(1, math.floor(L * 2 / (smax * (1 + 1e-4)))), 1 << 20)) for L in gbox])
    return lo, gbox / nc, nc


def _survey_chunk_catalogue(mode, seed, smax):
    """(sky columns, cells per axis): six cells of the survey grid hold exactly 127 .. 257 rows each (a clump, half of
    its rows duplicates), a background the other cells; the background's rows set the grid's extent"""
    rng = np.random.RandomState(seed)
    if mode == "angular":
        sky = so.sky_catalogue(seed, 700, ra=(20., 30.), dec=(10., 18.))
    else:
        sky = so.sky_catalogue(seed, 700, ra=(20., 40.), dec=(10., 25.), z=(0.05, 0.005))
    bg = _sky_rows(mode, *sky)
    lo, cs, nc = _survey_grid(bg, smax)
    assert (nc >= 6).all()
    f = (bg - lo) / cs
    idx = np.minimum(np.floor(f).astype(np.int64), nc - 1)
    frac = f - idx
    # clump centres: background rows well inside their cell and 2 cells inside the grid
    ok = ((frac > 0.3) & (frac < 0.7) & (idx >= 2) & (idx <= nc - 3)).all(1)
    keys = np.ravel_multi_index(tuple(idx.T), tuple(nc))
    cand = np.nonzero(ok)[0]
    _, first = np.unique(keys[cand], return_index=True)
    cand = cand[np.sort(first)]
    assert len(cand) >= len(_CELL_ROWS)
    centres = cand[:len(_CELL_ROWS)]
    parts = []
    for c, n in zip(centres, _CELL_ROWS):
        u = bg[c] + np.clip(rng.normal(scale=0.05, size=((n + 1) // 2, 3)), -0.15, 0.15) * cs
        if mode == "angular":
            u /= np.linalg.norm(u, axis=1)[:, None]
        parts.append(np.concatenate([u, u[:n // 2]]))
    # the background outside the clump cells, without rows within 1e-6 of a cell face (the sky round trip moves rows by
    # about 1e-9), but keeping the rows that set the grid's extent
    edge = ((bg == bg.min(0)) | (bg == bg.max(0))).any(1)
    near = ((frac < 1e-6) | (frac > 1 - 1e-6)).any(1)
    keep = edge | (~np.isin(keys, keys[centres]) & ~near)
    clumps = _to_sky(np.concatenate(parts), mode)
    if mode == "angular":
        return (np.concatenate([sky[0][keep], clumps[0]]), np.concatenate([sky[1][keep], clumps[1]]), None), nc
    return tuple(np.concatenate([a[keep], b]) for a, b in zip(sky, clumps)), nc


@pytest.mark.parametrize("mode", ["1d", "2d", "projected", "angular"])
def test_survey_cells_at_chunk_boundaries(grids, mode):
    """primary cells of exactly 127, 128, 129, 255, 256 and 257 rows, weighted auto counts"""
    if mode == "angular":
        edges, kw = np.linspace(0.005, 0.5, 6), {}
        smax = float(so.chord_edges(edges)[-1])
    else:
        edges = np.linspace(0.05, 8., 6)
        kw = dict(Nmu=5) if mode == "2d" else (dict(pimax=8.) if mode == "projected" else {})
        smax = math.sqrt(64. + 64.) if mode == "projected" else 8.
    seed = 320 + len(mode)
    sky, nc = _survey_chunk_catalogue(mode, seed, smax)
    w = np.random.RandomState(seed).uniform(0.5, 2., len(sky[0]))
    _survey(mode, sky, edges, w1=w, **kw)
    g = _checked(grids)[-1]                         # the primaries' grid, built after the secondaries'
    assert g["ncell"] == nc.tolist()
    _assert_cell_rows(g, int(_lib().nbk_paircount_chunk_rows()))


def _dyadic_pairs():
    """rows in pairs x1 = a e + c f, x2 = b e - c f for the axes e = +-x, +-y, +-z and a perpendicular axis f: the pair's
    line of sight l = x1 + x2 lies along e, so pi = b - a and r_p = 2c exactly"""
    rows, pis, axes = [], [], []
    for axis in range(3):
        for sign in (1., -1.):
            e = np.zeros(3)
            e[axis] = sign
            f = np.zeros(3)
            f[(axis + 1) % 3] = 1.
            for a, b in ((100., 132.), (140., 156.), (60., 92.)):
                for c in (1.5, 2.5, 3.25):
                    rows += [a * e + c * f, b * e - c * f]
                    pis.append(b - a)
                    axes.append(axis)
    return np.array(rows), np.array(pis), np.array(axes)


def test_survey_projected_pi_at_pimax(grids):
    """pimax = 32: pi exactly pimax is excluded; pimax one ulp above 32: pi = 32, one ulp below pimax, is included.  The
    pairs whose line of sight lies along x or y are 16 or 32 apart across the grid's columns, where a column gap above
    r_p,max would skip them, so only the sphere prune (s_max^2 = r_p,max^2 + pimax^2) visits them"""
    from nbodykit_b200.algorithms.paircount import count_pairs
    rows, pis, axes = _dyadic_pairs()
    edges = np.array([1., 4., 5.5, 7.])
    t = torch.from_numpy(rows).cuda()
    w = torch.from_numpy(np.random.RandomState(330).uniform(0.5, 2., len(rows))).cuda()
    total = []
    for pm in (32., float(np.nextafter(32., np.inf))):
        n, ws, ss, _ = count_pairs("projected", t, w, t, w, edges, False, None, pimax=pm, survey=True)
        want = so.brute_force(rows, "projected", edges, w1=w.cpu().numpy(), pimax=pm)
        shape = want["npairs"].shape
        np.testing.assert_array_equal(n.cpu().numpy().reshape(shape), want["npairs"])
        np.testing.assert_allclose(ws.cpu().numpy().reshape(shape), want["wnpairs"], rtol=1e-12, atol=0)
        np.testing.assert_allclose(ss.cpu().numpy().reshape(shape), want["sepsum"], rtol=1e-12, atol=0)
        total.append(int(want["npairs"].sum()))
    # the pairs with pi exactly 32, every constructed one among them in both orders, count only below the larger pimax
    assert total[1] - total[0] >= 2 * int((pis == 32.).sum()) > 0
    g = _checked(grids)[-1]                         # of the larger pimax
    cs = g["box"] / np.asarray(g["ncell"])
    cell = np.floor((rows - g["origin"]) / cs)
    delta = np.abs(cell[0::2] - cell[1::2])[np.arange(len(pis)), axes]
    gap = (delta - 1) * cs[axes] - g["tol"][axes]
    # pairs with pi = 32 along x or y, counted below the larger pimax, whose columns lie beyond r_p,max
    assert ((axes < 2) & (pis == 32.) & (gap > edges[-1])).sum() >= 6


@pytest.mark.parametrize("dtype", ["f4", "f8"])
@pytest.mark.parametrize("mode", ["1d", "2d", "projected"])
def test_survey_thin_shell_far_from_observer(grids, mode, dtype):
    """a shell 3000 < r < 3010 Mpc/h on a 3 x 3 degree patch: the grid's origin is hundreds of cells from the observer,
    so the tolerance 4e-7 (box + |origin|) of a row outside its cell is set by |origin|"""
    rng = np.random.RandomState(340)
    n = 3000
    ra, dec = np.deg2rad(rng.uniform(10., 13., n)), np.deg2rad(rng.uniform(10., 13., n))
    r = rng.uniform(3000., 3010., n)
    rows = np.stack([r * np.cos(dec) * np.cos(ra), r * np.cos(dec) * np.sin(ra), r * np.sin(dec)], 1)
    sky = tuple(np.asarray(a, dtype) for a in _to_sky(rows, mode))
    w = rng.uniform(0.5, 2., n)
    kw = dict(Nmu=6) if mode == "2d" else (dict(pimax=5.) if mode == "projected" else {})
    _survey(mode, sky, np.linspace(0.5, 6., 6), w1=w, dtype=dtype, **kw)
    g = _checked(grids)[-1]                         # the primaries' grid, built after the secondaries'
    cs = g["box"] / np.asarray(g["ncell"])
    assert np.linalg.norm(g["origin"]) > 2500. and (np.abs(g["origin"]) > 100 * cs).any()
    assert (g["tol"] > 4e-7 * g["box"] * 10).any()


def test_survey_angular_to_180_degrees_antipodal_and_coincident(grids):
    """theta edges up to 180 degrees (one cell per axis), antipodal and near-antipodal rows, coincident rows"""
    rng = np.random.RandomState(350)
    n = 400
    ra = rng.uniform(0., 360., n)
    dec = np.rad2deg(np.arcsin(rng.uniform(-1., 1., n)))
    ra = np.concatenate([ra, (ra[:40] + 180.) % 360., (ra[40:70] + 179.7) % 360., ra[70:100], [0., 180., 90., 270.]])
    dec = np.concatenate([dec, -dec[:40], -dec[40:70], dec[70:100], [0., 0., 90., -90.]])
    edges = np.array([1., 60., 120., 179., 180.])
    r, want = _survey("angular", (ra, dec, None), edges, w1=rng.uniform(0.5, 2., len(ra)), brute=True)
    assert want["npairs"][-1] >= 2 * 30
    g = _checked(grids)[-1]                         # the primaries' grid, built after the secondaries'
    assert g["ncell"] == [1, 1, 1]


# ---- CylindricalGroups --------------------------------------------------------------------------------------------------
def _cgm(pos, key, rperp, rpar, los=None, periodic=False, box=None):
    """CylindricalGroups ranked by `key` against the oracle: the three columns bit for bit, and the number of directed
    links to a higher-priority row equal to the length of the neighbour lists the count and write passes built"""
    from nbodykit_b200.lab import ArrayCatalog, CylindricalGroups
    data = {"Position": torch.as_tensor(np.ascontiguousarray(pos)).cuda(), "k": torch.from_numpy(key).cuda()}
    kw = dict(BoxSize=np.ones(3) * np.asarray(box, "f8")) if periodic else {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        r = CylindricalGroups(ArrayCatalog(data, comm=_comm(), **kw), "k", rperp, rpar, flat_sky_los=los,
                              periodic=periodic)
    t, h, s, prio = co.cgm(pos, [key], rperp, rpar, los=los, periodic=periodic, BoxSize=box)
    np.testing.assert_array_equal(np.asarray(r.groups["cgm_type"].compute()), t)
    np.testing.assert_array_equal(np.asarray(r.groups["cgm_haloid"].compute()), h)
    np.testing.assert_array_equal(np.asarray(r.groups["num_cgm_sats"].compute()), s)
    L = np.ones(3) * np.asarray(box, "f8") if periodic else None
    x = (co.wrap(np.asarray(pos), L) if periodic else np.asarray(pos)).astype("f8")
    i, j = co.candidates(x, math.sqrt(rperp * rperp + rpar * rpar), L)
    hi, lo = np.where(prio[i] > prio[j], i, j), np.where(prio[i] > prio[j], j, i)
    links = int(co.linked(x[hi], x[lo], rperp, rpar, los, L).sum())
    assert r._stats["neighbours"] == links
    assert links > 0 and 0 < int((t == 1).sum()) < len(pos)
    return r, x[hi], x[lo]


@pytest.mark.parametrize("L", [L_UP, L_DOWN], ids=["Lf4_above_L", "Lf4_below_L"])
def test_cgm_box_side_not_exact_in_f4(grids, L):
    rng = np.random.RandomState(400)
    pos = np.concatenate([(rng.uniform(size=(2500, 3)) * L).astype("f4"), _edge_rows(rng, L, 250)])
    _assert_wraps_onto_L_f4(pos, L)
    key = rng.uniform(size=len(pos))
    _cgm(pos, key, 2.5, 4., los=[0, 0, 1], periodic=True, box=L)
    (g,) = _checked(grids)
    assert (g["pos"] == _f4(L)).any()


@pytest.mark.parametrize("los", [None, [0.6, 0.8, 0.]], ids=["observer", "flat"])
def test_cgm_noncubic_periodic_box(grids, los):
    box = np.array([30., 45., 60.])
    rng = np.random.RandomState(401)
    pos = np.concatenate([rng.uniform(size=(3000, 3)) * box, [[0., 0., 0.], box - 1e-9, [-1e-9, 22.5, 60.]]])
    key = rng.randint(0, 50, len(pos)).astype("f8")
    _cgm(pos, key, 2., 3., los=los, periodic=True, box=box)
    (g,) = _checked(grids)
    assert len(set(g["ncell"])) == 3


@pytest.mark.parametrize("cells", [1, 2, 3])
def test_cgm_sparse_widened_to_few_cells(grids, cells):
    """54, 250 and 686 rows in a periodic box of 8 cells per axis at rmax / 2: the widening to about 16 rows per cell
    leaves 1, 2 and 3 cells per axis, where the stencil visits every cell once"""
    L, rperp, rpar = 30., 4., 6.
    n = {1: 54, 2: 250, 3: 686}[cells]
    rng = np.random.RandomState(402 + cells)
    pos = np.concatenate([rng.uniform(size=(n - 3, 3)) * L, [[0., 0., 0.], [L - 1e-9] * 3, [-1e-9, L / 2, 1e-9]]])
    key = rng.uniform(size=n)
    _cgm(pos, key, rperp, rpar, los=[0, 0, 1], periodic=True, box=L)
    (g,) = _checked(grids)
    rmax = math.hypot(rperp, rpar)
    assert math.floor(2 * L / (rmax * 1.0001)) == 8
    assert g["ncell"] == [cells] * 3


def _zwrap_catalogue(seed):
    """4000 distinct rows on a lattice of 1.5 in x and y and of 60 z values, a third of them within 1 of a z face"""
    rng = np.random.RandomState(seed)
    xy = np.arange(14) * 1.5 + 0.25
    zs = np.concatenate([np.sort(rng.uniform(0., 100., 40)), rng.uniform(0., 1., 10), 100. - rng.uniform(0., 1., 10)])
    idx = rng.choice(14 * 14 * 60, size=4000, replace=False)
    i, j, k = np.unravel_index(idx, (14, 14, 60))
    return np.stack([xy[i], xy[j], zs[k]], 1)


@pytest.mark.parametrize("rperp,rpar", [(2., 3.), (0., 3.), (2., 0.)])
def test_cgm_z_reach_wraps_at_both_faces(grids, rperp, rpar):
    """a periodic box of 20 x 20 x 100 widened to 3 x 3 x 18 cells: x and y visited whole, and the z reach of the cells
    next to both z faces split into two wrapped ranges; rperp = 0 links rows of one (x, y) column, rpar = 0 rows of one
    z plane"""
    box = np.array([20., 20., 100.])
    pos = _zwrap_catalogue(410)
    key = np.random.RandomState(411).uniform(size=len(pos))
    r, xa, xb = _cgm(pos, key, rperp, rpar, los=[0, 0, 1], periodic=True, box=box)
    (g,) = _checked(grids)
    assert g["ncell"] == [3, 3, 18]
    cs = box / np.asarray(g["ncell"])
    reach = [math.floor((math.hypot(rperp, rpar) * (1 + 1e-9) + 2 * t) / c * (1 + 1e-12)) + 1 for t, c in zip(g["tol"], cs)]
    assert [2 * r_ + 1 >= c for r_, c in zip(reach, g["ncell"])] == [True, True, False]
    # links across the faces: in z from the first and the last z cell (rpar = 0 links rows of one z plane only, across
    # the x and y faces)
    across = np.abs(xa - xb) > box / 2
    assert across[:, 2 if rpar > 0 else 0].sum() > 10


def _cgm_chunk_catalogue(seed, L, nc):
    """cells of exactly 127 .. 257 rows (a tight clump in each, half of its rows duplicates) and a background in the
    other cells, on the periodic grid of nc cells per axis"""
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


@pytest.mark.parametrize("los", [None, [0, 0, 1]], ids=["observer", "flat"])
def test_cgm_cells_at_chunk_boundaries(grids, los):
    """cells of 127 .. 257 rows, keys with 4 values so that priorities tie and go by row across every chunk boundary;
    the count and the write pass must list the same links"""
    from nbodykit_b200._lib import lib
    L, rperp, rpar = 40., 10., 15.
    nc = math.floor(2 * L / (math.hypot(rperp, rpar) * 1.0001))
    assert nc == 4
    pos = _cgm_chunk_catalogue(420, L, nc)
    assert len(pos) >= 16 * nc ** 3                 # no widening
    key = np.random.RandomState(421).randint(0, 4, len(pos)).astype("f8")
    _cgm(pos, key, rperp, rpar, los=los, periodic=True, box=L)
    (g,) = _checked(grids)
    assert g["ncell"] == [nc] * 3
    _assert_cell_rows(g, int(lib().nbk_cgm_chunk_rows()))


@pytest.mark.parametrize("los", [None, [0, 0, 1]], ids=["observer", "flat"])
def test_cgm_far_from_origin_f4(grids, los):
    rng = np.random.RandomState(430)
    p = np.concatenate([rng.uniform(size=(1500, 3)) * 30., rng.normal(scale=1.5, size=(1500, 3)) + 15.])
    pos = (p + np.array([1e5, -4e5, 1e6])).astype("f4")
    _cgm(pos, rng.uniform(size=len(pos)), 0.6, 1.2, los=los)
    (g,) = _checked(grids)
    assert np.all(np.abs(g["origin"]) > 9e4)


@pytest.mark.parametrize("shape", ["plane", "line"])
def test_cgm_nonperiodic_plane_and_line(grids, shape):
    """all z equal, or all rows on a line along x: the grid takes a side of 1 where hi == lo"""
    rng = np.random.RandomState(431)
    if shape == "plane":
        pos = rng.uniform(size=(2000, 3)) * 30.
        pos[:, 2] = 3.7
        los = [0.6, 0., 0.8]
    else:
        pos = np.zeros((800, 3)) + [1.5, -2.25, 8.]
        pos[:, 0] = rng.uniform(size=800) * 200.
        los = [1., 0., 0.]
    _cgm(pos, rng.uniform(size=len(pos)), 0.5, 0.8, los=los)
    (g,) = _checked(grids)
    for d in ([2] if shape == "plane" else [1, 2]):
        assert g["box"][d] == 1.


# ---- KDDensity -----------------------------------------------------------------------------------------------------------
def _kd(pos, L):
    from nbodykit_b200.lab import ArrayCatalog, KDDensity
    r = KDDensity(ArrayCatalog({"Position": torch.as_tensor(np.ascontiguousarray(pos)).cuda()}, comm=_comm(), BoxSize=L))
    d, dens = ko.density(pos, L)
    np.testing.assert_array_equal(r._distance, d)
    np.testing.assert_allclose(r.density, dens, rtol=1e-15, atol=0)
    return r, d


@pytest.mark.parametrize("c", range(2, 11))
def test_kd_cell_count_at_row_boundaries(grids, c):
    """N = 4 c^3 - 1 rows give c - 1 cells per axis and N = 4 c^3 give c (the (1 + 1e-12) of _ncell lifts the cube
    root, e.g. 500 rows give 5)"""
    rng = np.random.RandomState(440 + c)
    for N, want in ((4 * c ** 3 - 1, c - 1), (4 * c ** 3, c)):
        r, _ = _kd(rng.uniform(size=(N, 3)) * 50., 50.)
        assert r._stats["ncell"] == want
        assert _checked(grids)[-1]["ncell"] == [want] * 3


def _kd_grid_offsets(nc):
    lo = (nc - 1) // 2
    return lo, nc - 1 - lo


@pytest.mark.parametrize("nc", [4, 5, 6])
def test_kd_neighbours_only_in_last_ring(grids, nc):
    """7 rows in cell (0, 0, 0) and the rest in cells nc // 2 .. away on every axis: the 8th neighbour of the 7 lies in
    the last ring of the walk, at offset +hi (even nc, where -lo .. hi is asymmetric) or at both +-2 (nc = 5)"""
    lo, hi = _kd_grid_offsets(nc)
    assert (hi == lo + 1) == (nc % 2 == 0)
    rng = np.random.RandomState(450 + nc)
    cs = 1. / nc
    N = 4 * nc ** 3 + 10
    group = (0.5 + rng.uniform(-0.05, 0.05, size=(7, 3))) * cs
    far = [hi] if nc % 2 == 0 else [hi, nc - lo]
    bulk = []
    for k, c in enumerate(far):
        m = (N - 7) // len(far) + (N - 7) % len(far) * (k == 0)
        bulk.append((c + rng.uniform(0.1, 0.9, size=(m, 3))) * cs)
    pos = np.concatenate([group] + bulk)
    r, d = _kd(pos, 1.)
    assert len(pos) == N and r._stats["ncell"] == nc
    # only the 7 rows lie within ring hi - 1 of cell (0, 0, 0); their 8th neighbour does not
    cell = np.floor(pos / cs).astype(int)
    off = np.minimum(cell, nc - cell).max(1)
    assert (off < hi).sum() == 7 and np.isfinite(d[:7]).all()
    assert (d[:7] > (hi - 1) * cs).all()
    _checked(grids)


@pytest.mark.parametrize("nc", [4, 5, 8])
def test_kd_rows_on_cell_faces(grids, nc):
    """4 copies of every lattice point q = k / nc (N = 4 nc^3): every row lies on a cell face, and its 8th distance is
    one cell side, the lower bound of the ring beyond its neighbours"""
    k = np.arange(nc) / nc
    lat = np.stack(np.meshgrid(k, k, k, indexing="ij"), -1).reshape(-1, 3)
    pos = np.concatenate([lat] * 4)
    r, d = _kd(pos, 1.)
    assert r._stats["ncell"] == nc
    np.testing.assert_allclose(d, 1. / nc, rtol=1e-15)
    if nc in (4, 8):
        assert (d == 1. / nc).all()
    _checked(grids)


@pytest.mark.parametrize("L", [L_UP, L_DOWN], ids=["Lf4_above_L", "Lf4_below_L"])
def test_kd_box_side_not_exact_in_f4(grids, L):
    """float32 rows at L_f4, one ulp below it and just below 0, where q = f4(x / L) % 1 rounds to 1.0 and becomes 0"""
    rng = np.random.RandomState(460)
    pos = np.concatenate([(rng.uniform(size=(3000, 3)) * L).astype("f4"), _edge_rows(rng, L, 300)])
    _kd(pos, L)
    q = ko.unit(pos, L)
    assert ((pos < 0) & (q == 0)).any()
    assert (pos == np.float32(L)).any()
    _checked(grids)


# ---- FiberCollisions -----------------------------------------------------------------------------------------------------
def _fc(ra, dec, collision_radius, seed=7):
    """FiberCollisions against the oracle; returns the run, the float32 positions and the three columns"""
    from nbodykit_b200.lab import FiberCollisions
    r = FiberCollisions(ra, dec, collision_radius=collision_radius, seed=seed, comm=_comm())
    lab, col, nb = [np.asarray(r.labels[c].compute()) for c in ("Label", "Collided", "NeighborID")]
    pos = r.source["Position"].compute().cpu().numpy()
    want = fo.fiber_collisions(pos, r._collision_radius_rad, seed)
    np.testing.assert_array_equal(lab, want[0])
    np.testing.assert_array_equal(col, want[1])
    np.testing.assert_array_equal(nb, want[2])
    return r, pos.astype("f4"), lab, col, nb


def _fc_cells(rad):
    """the cells of FiberCollisions' larger groups: nc = floor(2.2 / (rad (1 + 1e-6))) per axis"""
    nc = max(1, int(math.floor(2.2 / (rad * (1 + 1e-6)))))
    return nc, 2.2 / nc


_FC_SIZES = [2, 3, 31, 32, 33, 2048, 2049]


def _fc_layout(layout, rad_deg):
    """one chain (or two-wide ladder) group of each size in _FC_SIZES, members 0.7 (ladder: 0.75) radii apart"""
    ra, dec = [], []
    for k, n in enumerate(_FC_SIZES):
        d0 = -6. + 1.5 * k
        if layout == "chain":
            a = 0.7 * rad_deg
            ra.append(100. + np.arange(n) * a / math.cos(math.radians(d0)))
            dec.append(np.full(n, d0))
        else:
            a = 0.75 * rad_deg
            m = np.arange(n)
            ra.append(100. + (m // 2) * a / math.cos(math.radians(d0)))
            dec.append(d0 + (m % 2) * a)
    return np.concatenate(ra), np.concatenate(dec)


@pytest.mark.parametrize("layout", ["chain", "ladder"])
def test_fc_group_sizes_around_the_greedy_paths(cuda, layout):
    """groups of 2 (pairs), 3, 31, 32 (one warp), 33, 2048 (a block in shared memory) and 2049 members (global scratch)
    in one catalogue; the long groups straddle many faces of the cell grid"""
    rad_deg = 62 / 3600.
    ra, dec = _fc_layout(layout, rad_deg)
    perm = np.random.RandomState(470).permutation(len(ra))
    r, p4, lab, col, nb = _fc(ra[perm], dec[perm], rad_deg)
    assert int(_lib().nbk_fc_warp_members()) == 32 and int(_lib().nbk_fc_smem_members()) == 2048
    sizes = np.bincount(lab)[1:]
    assert sorted(sizes.tolist()) == _FC_SIZES
    assert r._stats["largest"] == 2049 and r._stats["pairs"] == 1
    fo.check_invariants(p4, lab, col, nb, r._collision_radius_rad)
    nc, cs = _fc_cells(r._collision_radius_rad)
    big = lab == np.argmax(np.bincount(lab))
    cells = np.floor(p4[big].astype("f8") / cs)
    assert len(np.unique(cells[:, 1])) > 5 and len(np.unique(cells[:, 0])) > 1


def _tie_offset(k):
    """t such that float32(1.1 + t) and float32(1.1 - t) lie k float32 ulps either side of float32(1.1)"""
    c = np.float32(1.1)
    ulp = float(np.spacing(c))
    return float(c) + k * ulp - 1.1


@pytest.mark.parametrize("first", ["A", "B", "N1"])
@pytest.mark.parametrize("path", ["warp", "block"])
def test_fc_nearest_member_ties(cuda, path, first):
    """C at (ra, dec) = (0, 0) collides with A and B at ra = +-a and with the first row N1 of a chain going north; it is
    removed first, and A, B (and N1 when uncollided) are at exactly the same float32 distance from it.  The first of them
    in member order must win, in the warp path (9 members) and in the ring walk of the block path (43 members), whichever
    of them holds the lowest row"""
    t = _tie_offset(2500)
    a = math.degrees(math.asin(t))
    M = 6 if path == "warp" else 40
    rows = {"A": (a, 0.), "B": (-a, 0.), "C": (0., 0.)}
    rows.update({"N%d" % k: (0., k * a) for k in range(1, M + 1)})
    order = [first] + [k for k in ["A", "B", "N1", "C"] if k != first] + ["N%d" % k for k in range(2, M + 1)]
    ra = np.array([rows[k][0] for k in order])
    dec = np.array([rows[k][1] for k in order])
    r, p4, lab, col, nb = _fc(ra, dec, 1.3 * a)
    assert len(set(lab.tolist())) == 1 and lab[0] > 0 and len(lab) == M + 3
    assert (M + 3 > 32) == (path == "block")
    i = {k: order.index(k) for k in ("A", "B", "C", "N1")}
    d = {k: fo._dist(p4[i["C"]], p4[i[k]]) for k in ("A", "B", "N1")}
    assert d["A"] == d["B"] == d["N1"]
    assert col[i["C"]] == 1 and col[i["A"]] == 0 and col[i["B"]] == 0
    tied = sorted(i[k] for k in ("A", "B", "N1") if col[i[k]] == 0)
    assert len(tied) >= 2 and nb[i["C"]] == tied[0]


@pytest.mark.parametrize("nc", [1, 2, 3])
def test_fc_large_radius_few_cells(cuda, nc):
    """collision radii of 1.2, 0.8 and 0.6 rad: 1, 2 and 3 cells per axis, so the 3 x 3 x 3 lists and the ring walk are
    clamped on both sides; 60 rows over the whole sky make a group above one warp"""
    rad = {1: 1.2, 2: 0.8, 3: 0.6}[nc]
    assert _fc_cells(rad)[0] == nc
    rng = np.random.RandomState(480 + nc)
    ra = rng.uniform(0., 360., 60)
    dec = np.rad2deg(np.arcsin(rng.uniform(-1., 1., 60)))
    r, p4, lab, col, nb = _fc(ra, dec, math.degrees(rad))
    assert _fc_cells(r._collision_radius_rad)[0] == nc
    assert np.bincount(lab)[1:].max() > 32
    fo.check_invariants(p4, lab, col, nb, r._collision_radius_rad)


def _degrees_for(rad, above):
    """a collision radius in degrees whose numpy.deg2rad is rad, else the nearest one above (or below) it"""
    c0 = math.degrees(rad)
    cands = [c0]
    for d in (np.inf, -np.inf):
        c = c0
        for _ in range(16):
            c = float(np.nextafter(c, d))
            cands.append(c)
    got = [(float(np.deg2rad(c)), c) for c in cands]
    exact = [c for v, c in got if v == rad]
    if exact:
        return exact[0]
    side = [(abs(v - rad), c) for v, c in got if (v > rad) == above]
    return min(side)[1]


@pytest.mark.parametrize("side", ["below", "equal", "above"])
def test_fc_pair_at_the_radius(cuda, side):
    """A and B a float32 distance D apart with C between them: rad = D (1 - 1e-12), D and D (1 + 1e-12).  A and B collide
    from D on, and the greedy then removes two of the three instead of C alone"""
    from nbodykit_b200 import transform as T
    ra = np.array([10., 10.02, 10.01] + list(np.linspace(50., 60., 20)))
    dec = np.array([5., 5.003, 5.0015] + list(np.linspace(-20., -10., 20)))
    p = (T.SkyToUnitSphere(torch.from_numpy(ra).cuda(), torch.from_numpy(dec).cuda()) + 1.1).cpu().numpy().astype("f4")
    D = float(fo._dist(p[0], p[1]))
    target = D * {"below": 1 - 1e-12, "equal": 1., "above": 1 + 1e-12}[side]
    r, p4, lab, col, nb = _fc(ra, dec, _degrees_for(target, above=side != "below"))
    np.testing.assert_array_equal(p4, p)
    rad = r._collision_radius_rad
    assert abs(rad - target) <= 5e-16 * target
    assert abs(D - rad) <= 1.01e-12 * rad and (D <= rad) == (side != "below")
    assert lab[0] == lab[1] == lab[2] > 0 and np.bincount(lab)[lab[0]] == 3
    assert col[:3].sum() == (1 if side == "below" else 2)


# ---- several ranks ---------------------------------------------------------------------------------------------------
def _slab_rows(P, seed):
    """inputs of every algorithm with rows on the x-slab boundaries of P ranks"""
    rng = np.random.RandomState(seed)
    out = {}
    # survey 'projected': Cartesian rows, some on the boundaries of P equal slabs of their x extent (to the 1e-9 of the
    # sky round trip), as sky columns
    cart = np.stack([rng.uniform(100., 160., 1500), rng.uniform(-30., 30., 1500), rng.uniform(50., 110., 1500)], 1)
    lo, hi = 100., 160.
    cart[0, 0], cart[1, 0] = lo, hi
    for k in range(1, P):
        cart[k * 40:(k + 1) * 40, 0] = lo + k * (hi - lo) / P
    out["survey"] = _to_sky(cart, "projected")
    out["survey_w"] = rng.uniform(0.5, 2., len(cart))
    # CylindricalGroups and KDDensity in periodic boxes whose slab boundaries are k L / P
    L = 30.
    pos = rng.uniform(size=(3000, 3)) * L
    for k in range(P):
        pos[k * 50:(k + 1) * 50, 0] = k * L / P
    pos[-20:, 0] = L - 1e-9
    out["cgm"] = pos
    out["cgm_key"] = rng.randint(0, 20, len(pos)).astype("f8")
    out["kd"] = (pos / L * 6.).copy()
    # FiberCollisions: clumps on the x-slab boundaries of the FOF box 2.2 (x = cos(dec) cos(ra) + 1.1)
    ra, dec = [rng.uniform(0., 360., 1500)], [np.rad2deg(np.arcsin(rng.uniform(-1., 1., 1500)))]
    for k in range(1, P):
        cx = 2.2 * k / P - 1.1
        r0, d0 = math.degrees(math.acos(cx / math.cos(math.radians(10.)))), 10.
        ra.append(r0 + rng.normal(scale=0.01, size=60))
        dec.append(d0 + rng.normal(scale=0.01, size=60))
    out["fc"] = (np.concatenate(ra), np.concatenate(dec))
    return out


def _all_ranks(comm, data, split):
    """rank r runs every algorithm on rows [split[name][r], split[name][r + 1]) of each input"""
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200.lab import ArrayCatalog, CylindricalGroups, FiberCollisions, KDDensity, SurveyDataPairCount

    def mine(name):
        return slice(split[name][comm.rank], split[name][comm.rank + 1])
    s = mine("survey")
    sk = data["survey"]
    r = SurveyDataPairCount("projected", _sky_cat(sk[0][s], sk[1][s], sk[2][s], data["survey_w"][s], comm=comm),
                            np.linspace(1., 12., 5), cosmo=Planck15, pimax=10.)
    out = dict(npairs=r.pairs["npairs"], wnpairs=r.pairs["wnpairs"], rp=r.pairs["rp"])
    s = mine("cgm")
    cat = ArrayCatalog({"Position": torch.from_numpy(data["cgm"][s]).cuda(), "k": torch.from_numpy(data["cgm_key"][s]).cuda()},
                       comm=comm, BoxSize=[30.] * 3)
    g = CylindricalGroups(cat, "k", 1.5, 2.5, flat_sky_los=[0, 0, 1], periodic=True)
    out.update({c: np.asarray(g.groups[c].compute()) for c in ("cgm_type", "cgm_haloid", "num_cgm_sats")})
    kd = KDDensity(ArrayCatalog({"Position": torch.from_numpy(data["kd"][s]).cuda()}, comm=comm, BoxSize=6.))
    out["kd"] = kd._distance
    s = mine("fc")
    f = FiberCollisions(data["fc"][0][s], data["fc"][1][s], collision_radius=0.05, seed=3, comm=comm)
    out.update({c: np.asarray(f.labels[c].compute()) for c in ("Label", "Collided", "NeighborID")})
    return out


@pytest.mark.parametrize("P", [2, 3])
def test_several_ranks_rows_on_slab_boundaries(cuda, P):
    """P gloo ranks sharing device 0, one of them empty for P = 3, reproduce the one-rank answer of every algorithm"""
    from test_gpu_fof import _spawn
    data = _slab_rows(P, 490 + P)

    def split(n):
        if P == 3:
            return [0, 0, n // 3, n]
        return [0, n // 2, n]
    sp = {k: split(len(v[0]) if k in ("survey", "fc") else len(v)) for k, v in data.items() if k in ("survey", "cgm", "fc")}
    parts = _spawn(_all_ranks, P, data, sp)
    sk = data["survey"]
    want = so.count(_sky_rows("projected", *sk), "projected", np.linspace(1., 12., 5), w1=data["survey_w"], pimax=10.)
    for p in parts:
        np.testing.assert_array_equal(p["npairs"], want["npairs"])
        np.testing.assert_allclose(p["wnpairs"], want["wnpairs"], rtol=1e-12, atol=0)
    assert want["npairs"].sum() > 1000
    t, h, s, _ = co.cgm(data["cgm"], [data["cgm_key"]], 1.5, 2.5, los=[0, 0, 1], periodic=True, BoxSize=30.)
    for c, w in (("cgm_type", t), ("cgm_haloid", h), ("num_cgm_sats", s)):
        np.testing.assert_array_equal(np.concatenate([p[c] for p in parts]), w)
    assert 0 < int((t == 1).sum()) < len(t)
    np.testing.assert_array_equal(np.concatenate([p["kd"] for p in parts]), ko.distance(data["kd"], 6.))
    from nbodykit_b200 import transform as T
    ra, dec = data["fc"]
    pos = (T.SkyToUnitSphere(torch.from_numpy(ra).cuda(), torch.from_numpy(dec).cuda()) + 1.1).cpu().numpy()
    lab, col, nb = fo.fiber_collisions(pos, float(np.deg2rad(0.05)), 3)
    for c, w in (("Label", lab), ("Collided", col), ("NeighborID", nb)):
        np.testing.assert_array_equal(np.concatenate([p[c] for p in parts]), w)
    assert np.bincount(lab)[1:].max() > 32
    # the rows set on the boundaries are there, and the FOF box's x of the clumps is within 1e-3 of them
    for k in range(1, P):
        b = 2.2 * k / P
        assert (np.abs(pos[:, 0] - b) < 1e-3).sum() >= 30
        assert (data["cgm"][:, 0] == k * 30. / P).sum() == 50
