"""ConvolvedFFT3PCF on the GPU: the tile-listed Gram against NumPy and the dense Gram; the estimator against the float64
oracle (tests/convfft3pcf_oracle.py) in f8 and f4, CIC and interlaced TSC, on power-of-two, mixed-radix and Bluestein
meshes with spherical and wedge windows; the exact link to SimulationBox3PCF(periodic=False) on grid-node objects;
the oracle's direct form over true separations in a box at the geometry guard's threshold, interlaced or not; 'c16' / 'c8' against 'f8' / 'f4'; the blocked
path; P = 2, 3, 4 ranks sharing one GPU against one rank.  tests/mgpu_check_convfft3pcf.py runs the several-GPU
comparison under torchrun.

Tolerances: nsep is an integer count and must match exactly; |d nnn_l| <= tol * bound_l(N) and |d rrr_l| <= tol *
bound_l(Rf) with bound_l(W) = (2l + 1) / (16 pi^2) sum_x |W| (sum_{s1} |W|) (sum_{s2} |W|), tol = 1e-10 (f8) or 1e-4
(f4); zeta is exactly threeptcf.edge_correct of the reported nnn and rrr."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import convfft3pcf_oracle as cfo
from test_gpu_bispectrum import SHAPES, TOL

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLES = [0, 1, 2, 3, 4]
NBAR = 1e-3


def _ball(rng, n, radius, wedge=False):
    """n points uniform in a ball (wedge: only x > 0 and y > |z|) about the origin"""
    out = np.zeros((0, 3))
    while len(out) < n:
        p = rng.uniform(-radius, radius, (4 * n, 3))
        ok = (p ** 2).sum(1) < radius ** 2
        if wedge:
            ok &= (p[:, 0] > 0) & (p[:, 1] > np.abs(p[:, 2]))
        out = np.concatenate([out, p[ok]])
    return out[:n]


def _columns(C, radius, seed, nd=800, nr=4000, wedge=False):
    """data (a clumpy sample) and randoms (10x denser, uniform) in a ball or wedge of `radius` about C"""
    rng = np.random.RandomState(seed)
    d = _ball(rng, nd, radius, wedge)
    d[:nd // 5] = d[:nd // 5] * 0.2 + d[nd // 5:2 * (nd // 5)] * 0.8     # clumps: a non-Gaussian field
    cats = {}
    for name, pos in (("data", d), ("randoms", _ball(rng, nr, radius, wedge))):
        n = len(pos)
        cats[name] = dict(Position=pos + C, Weight=rng.uniform(0.8, 1.2, n) if name == "data" else np.ones(n),
                          FKPWeight=rng.uniform(0.5, 1.0, n), NZ=np.full(n, NBAR))
    return cats


def _fkp(cats, comm=None, owner=None):
    from nbodykit_b200.lab import ArrayCatalog, FKPCatalog
    kw = {} if comm is None else dict(comm=comm)
    sp = []
    for name in ("data", "randoms"):
        cols = cats[name]
        mine = slice(None) if owner is None else owner[name] == comm.rank
        sp.append(ArrayCatalog({k: torch.from_numpy(np.ascontiguousarray(v[mine])).cuda() for k, v in cols.items()}, **kw))
    return FKPCatalog(sp[0], sp[1])


def _run(cats, N, L, C, dtype="f8", resampler="cic", interlaced=False, comm=None, owner=None, poles=POLES, edges=None):
    from nbodykit_b200.lab import ConvolvedFFT3PCF
    mesh = _fkp(cats, comm, owner).to_mesh(Nmesh=N, BoxSize=L, BoxCenter=C, dtype=dtype, resampler=resampler,
                                           interlaced=interlaced)
    return ConvolvedFFT3PCF(mesh, poles, edges)


def _geom(shape, support=3):
    """the shape's mesh, an off-origin centre, r_max and the largest ball radius the guard accepts (with a margin)"""
    N, L = SHAPES[shape]
    L = np.asarray(L, dtype="f8")
    H = L / np.asarray(N)
    rmax = 0.2 * L.min()
    radius = 0.45 * (L - (support + 2) * H - rmax).min()
    return N, L, np.array([350., -820., 1240.]), rmax, radius


def _raw_fields(r):
    """N and Rf from the call's own species paints (downloaded), before the window box"""
    mesh = r.first
    D = mesh["data"].to_real_field(normalize=False).numpy().astype("f8")
    R = mesh["randoms"].to_real_field(normalize=False).numpy().astype("f8")
    vc = float(np.prod(np.asarray(r.attrs["BoxSize"]) / np.asarray(r.attrs["Nmesh"])))
    a = r.attrs["alpha"]
    return (D - a * R) / vc, a * R / vc


def _masks(r):
    from nbodykit_b200.algorithms.convfft3pcf import box_mask
    return box_mask(r.attrs["Nmesh"], r.attrs["BoxSize"], *r.window)


def _boxed(r, fields):
    mx, my, mz = _masks(r)
    m = mx[:, None, None] * my[None, :, None] * mz[None, None, :]
    return tuple(f * m for f in fields)


def _fields(r):
    """N and Rf as the call sums them: its own paints, zero outside the window box"""
    return _boxed(r, _raw_fields(r))


def _unwrapped(r, *fields):
    """the fields rolled so that the window box starts at cell 0 on every axis: the oracle's direct form, which does
    not wrap, then sees the true separations of a survey painted across the index boundary"""
    out = []
    for f in fields:
        for ax, m in enumerate(_masks(r)):
            start = [i for i in range(len(m)) if m[i] and not m[i - 1]]
            assert len(start) == 1, "the window box is one interval shorter than the side"
            f = np.roll(f, -start[0], axis=ax)
        out.append(f)
    return out


def _stack(r, kind, poles=POLES):
    return np.stack([r.poles["%s_%d" % (kind, ell)] for ell in poles])


def _check(r, want, poles, tol, what):
    from nbodykit_b200.algorithms.threeptcf import edge_correct
    np.testing.assert_array_equal(r.nsep, want["nsep"], err_msg=what)
    for kind, bound in (("nnn", "bound_n"), ("rrr", "bound_r")):
        err = np.abs(_stack(r, kind, poles) - want[kind]) / want[bound]
        assert err.max() <= tol, "%s %s: |d| / bound = %.3g > %g" % (what, kind, err.max(), tol)
    z = edge_correct(_stack(r, "nnn", poles), _stack(r, "rrr", poles), poles)
    np.testing.assert_array_equal(_stack(r, "zeta", poles), z, err_msg=what)


# ---- the tile-listed Gram
def _gram(fn, w, A, na, B, nb, code, ncell, out, tiles=None):
    from nbodykit_b200 import _lib
    L = _lib.lib()
    if tiles is None:
        rc = L.nbk_fft3pcf_gram(w.data_ptr(), A.data_ptr(), A.shape[1], na, B.data_ptr(), B.shape[1], nb, code, ncell,
                                out.data_ptr(), None)
    else:
        rc = L.nbk_fft3pcf_gram_tiles(w.data_ptr(), A.data_ptr(), A.shape[1], na, B.data_ptr(), B.shape[1], nb, code,
                                      ncell, tiles.data_ptr() if tiles.numel() else None, tiles.numel(),
                                      out.data_ptr(), None)
    _lib.check(rc, fn)


@pytest.mark.parametrize("dtype", ["f8", "f4"])
@pytest.mark.parametrize("na,nb", [(1, 1), (5, 5), (32, 32), (7, 3), (32, 29)])
@pytest.mark.parametrize("which", ["empty", "full", "first", "last", "sparse"])
def test_listed_gram_matches_numpy_and_dense(cuda, dtype, na, nb, which):
    """w is zero outside the listed tiles; 20001 cells, so the last tile is partial"""
    from nbodykit_b200.algorithms.fft3pcf import GRAM_TILE
    rng = np.random.RandomState(na * 100 + nb)
    ncell = 20001
    ntile = -(-ncell // GRAM_TILE)
    tiles = {"empty": [], "full": list(range(ntile)), "first": [0], "last": [ntile - 1],
             "sparse": sorted(rng.choice(ntile, ntile // 3, replace=False))}[which]
    tdt = torch.float64 if dtype == "f8" else torch.float32
    code = 8 if dtype == "f8" else 4
    keep = np.zeros(ntile * GRAM_TILE, dtype=bool)
    for t in tiles:
        keep[t * GRAM_TILE:(t + 1) * GRAM_TILE] = True
    wh = np.where(keep[:ncell], rng.standard_normal(ncell), 0.)
    w = torch.from_numpy(wh).to(tdt).cuda()
    A = torch.from_numpy(rng.standard_normal((na, ncell + 3))).to(tdt).cuda()     # padded rows: stride != ncell
    B = torch.from_numpy(rng.standard_normal((nb, ncell + 3))).to(tdt).cuda()
    t = torch.tensor(np.asarray(tiles, dtype="i8"), dtype=torch.int64, device="cuda")
    wh, Ah, Bh = (x.cpu().numpy().astype("f8") for x in (w, A, B))
    for same in ([False, True] if na == nb else [False]):
        Bs, nbs, Bsh = (A, na, Ah) if same else (B, nb, Bh)
        got = torch.full((na, nbs), 1.5, dtype=torch.float64, device="cuda")        # accumulates
        dense = torch.full((na, nbs), 1.5, dtype=torch.float64, device="cuda")
        _gram("gram_tiles", w, A, na, Bs, nbs, code, ncell, got, t)
        _gram("gram", w, A, na, Bs, nbs, code, ncell, dense)
        want = 1.5 + (wh * Ah[:, None, :ncell] * Bsh[None, :, :ncell]).sum(-1)
        bound = 1.5 + (np.abs(wh) * np.abs(Ah[:, None, :ncell]) * np.abs(Bsh[None, :, :ncell])).sum(-1)
        g, d = got.cpu().numpy(), dense.cpu().numpy()
        mask = np.triu(np.ones((na, nbs), dtype=bool)) if same else np.ones((na, nbs), dtype=bool)
        assert (np.abs(g - want)[mask] <= 1e-12 * bound[mask]).all(), (which, same)
        assert (np.abs(g - d)[mask] <= 1e-12 * bound[mask]).all(), (which, same)
        if same:
            assert (g[~mask] == 1.5).all() and (d[~mask] == 1.5).all()
        if which == "empty":
            assert (g == 1.5).all()


def test_tile_list_marks_nonzero_tiles(cuda):
    from nbodykit_b200.algorithms.fft3pcf import GRAM_TILE, tile_list
    from nbodykit_b200.pmesh.pm import ParticleMesh, RealField
    pm = ParticleMesh(BoxSize=10., Nmesh=(9, 7, 5), dtype="f8")           # 315 cells: 5 tiles, the last partial
    f = RealField(pm)
    f[...] = 0.
    v = f.value.reshape(-1)
    v[3] = 1.
    v[314] = -2.
    v[2 * GRAM_TILE] = 1e-300
    assert tile_list(f).cpu().tolist() == [0, 2, 4]


# ---- the estimator
@pytest.mark.parametrize("window", [("cic", False), ("tsc", True)])
@pytest.mark.parametrize("dtype", ["f8", "f4"])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_matches_oracle(cuda, shape, dtype, window):
    N, L, C, rmax, radius = _geom(shape)
    cats = _columns(C, radius, 31, wedge=shape == "44x22x26")
    e = np.linspace(0, rmax, 5)
    r = _run(cats, N, L, C, dtype, *window, edges=e)
    raw = _raw_fields(r)
    Nf, Rf = _boxed(r, raw)
    want = cfo.fft_form(Nf, Rf, N, L, e, POLES)
    _check(r, want, POLES, TOL[dtype], "%s %s %s" % (shape, dtype, window))
    # the window's multipoles are far from zero: the edge correction is exercised
    assert (np.abs(want["rrr"][1:]) / want["bound_r"][1:]).max() > 1e-3
    assert r.poles.dims == ["r1", "r2"]
    assert r.poles.data.dtype.names == tuple("%s_%d" % (k, ell) for k in ("nnn", "rrr", "zeta") for ell in POLES)
    from nbodykit_b200.algorithms.fft3pcf import bin_blocks, transform_count
    assert r.attrs["transforms"] == transform_count(bin_blocks(4, 4), POLES, 2) == 2 + 3 * 4 * 25
    assert 0 < r.attrs["tiles"] < 0.9
    for key in ("poles", "edges", "Nmesh", "BoxSize", "BoxCenter", "alpha", "data.W", "randoms.W"):
        assert key in r.attrs
    d, rr = cats["data"], cats["randoms"]
    np.testing.assert_allclose(r.attrs["alpha"], d["Weight"].sum() / rr["Weight"].sum(), rtol=1e-12)
    if window[1]:
        # interlacing leaves band-limited tails outside the window box: the box cuts them
        assert np.abs(raw[0] - Nf).max() > 0
    else:
        # without interlacing the window box cuts nothing
        np.testing.assert_array_equal(raw[0], Nf)
        np.testing.assert_array_equal(raw[1], Rf)
        if dtype == "f8":
            # N is the FKP field FKPCatalogMesh.to_real_field paints
            F = r.first.to_real_field().numpy()
            np.testing.assert_allclose(Nf, F, rtol=0, atol=1e-12 * np.abs(F).max())


def test_direct_form_12(cuda):
    """independent of every FFT and of Y_lm: the oracle's direct sum over true separations at 12 x 10 x 9.  The
    survey sits in the middle of the mesh's cell index (recentred positions near L / 2), where the oracle's index
    separations are the true ones"""
    N, L, C = (12, 10, 9), np.array([120., 100., 90.]), np.array([40., 900., -300.])
    cats = _columns(C + L / 2, 12., 32, nd=200, nr=1000)
    e = np.array([5., 12., 19., 25.])
    r = _run(cats, N, L, C, "f8", "cic", edges=e)
    Nf, Rf = _fields(r)
    want = cfo.direct_form(Nf, Rf, N, L, e, POLES)
    _check(r, want, POLES, TOL["f8"], "direct")


def test_exact_link_to_simulationbox3pcf(cuda):
    """data and randoms on grid nodes (H = 2), painted with 'nnb': SimulationBox3PCF(periodic=False) on one row per
    nonzero node with weight N(x), and separately Rf(x), is the same sum as nnn_l and rrr_l, l = 0 .. 10.  The edges
    sit between the separations H sqrt(n)."""
    from nbodykit_b200.lab import ArrayCatalog, SimulationBox3PCF
    N, Lside = 32, 64.
    H = Lside / N
    L = np.array([Lside] * 3)
    C = np.array([200., -64., 32.])
    poles = list(range(11))
    e = H * np.sqrt(np.array([0.5, 4.5, 12.5, 30.5, 60.5, 100.5]))
    rng = np.random.RandomState(5)
    cats = {}
    for name, n, rad in (("data", 600, 8), ("randoms", 3000, 8)):
        k = np.rint(_ball(rng, n, rad)).astype("i8")
        if name == "data":
            k[:150] = k[:150] % 3 + 2                                # a clump
        cats[name] = dict(Position=k * H + C, Weight=np.ones(n), FKPWeight=rng.uniform(0.5, 1., n), NZ=np.full(n, NBAR))
    r = _run(cats, (N,) * 3, L, C, "f8", "nnb", poles=poles, edges=e)
    Nf, Rf = _fields(r)
    nodes = np.indices((N,) * 3).reshape(3, -1).T
    nodes = np.where(nodes < N // 2, nodes, nodes - N)                # the recentred node coordinates (-L/2, L/2]
    for kind, W, bk in (("nnn", Nf, "bound_n"), ("rrr", Rf, "bound_r")):
        w = W.reshape(-1)
        nz = w != 0
        cat = ArrayCatalog({"Position": torch.from_numpy(nodes[nz] * H).cuda(), "Weight": torch.from_numpy(w[nz]).cuda()},
                           BoxSize=L)
        ref = SimulationBox3PCF(cat, poles, e, periodic=False)
        want = np.stack([ref.poles["corr_%d" % ell] for ell in poles])
        bound = cfo._bound(W, cfo.fo.bins((N,) * 3, L, e), len(e) - 1, poles)
        err = np.abs(_stack(r, kind, poles) - want) / bound
        assert err.max() <= 1e-10, (kind, err.max())
        assert (np.abs(want[0]) / bound[0]).max() > 1e-3, kind
        assert (np.abs(want[1:]) / bound[1:]).max() > 1e-5, kind
        assert nz.sum() > 500


@pytest.mark.parametrize("window", [("cic", False), ("tsc", True)])
def test_direct_form_at_the_guard_threshold(cuda, window):
    """a survey centred on BoxCenter, so that it is painted across the index boundary of every axis, in a box 0.05 %
    above the smallest the guard accepts: the sums equal the oracle's direct form over true separations (no FFT, no
    wrap), interlaced or not"""
    from nbodykit_b200.algorithms.convfft3pcf import min_box_size
    from nbodykit_b200.pmesh.window import FindResampler
    N, C = (12, 12, 12), np.array([-310., 75., 905.])
    cats = _columns(C, 20., 38, nd=300, nr=1500)
    e = np.array([0., 10., 16., 20.])
    pos = np.concatenate([cats["data"]["Position"], cats["randoms"]["Position"]]) - C
    L = min_box_size(pos.min(0), pos.max(0), N, FindResampler(window[0]).support, e[-1]) * 1.0005
    r = _run(cats, N, L, C, "f8", *window, edges=e)
    Nf, Rf = _fields(r)
    for ax in range(3):
        assert np.abs(np.take(Nf, 0, axis=ax)).sum() > 0 and np.abs(np.take(Nf, N[ax] - 1, axis=ax)).sum() > 0
    Nu, Ru = _unwrapped(r, Nf, Rf)
    want = cfo.direct_form(Nu, Ru, N, L, e, POLES)
    assert (want["nsep"] > 0).all()
    _check(r, want, POLES, TOL["f8"], "threshold %s" % (window,))
    assert (np.abs(want["nnn"][0]) / want["bound_n"][0]).max() > 1e-3
    with pytest.raises(ValueError, match="BoxSize"):
        _run(cats, N, L * 0.999, C, "f8", *window, edges=e)


@pytest.mark.parametrize("cplx,real", [("c16", "f8"), ("c8", "f4")])
def test_complex_mesh_equals_real(cuda, cplx, real):
    N, L, C, rmax, radius = _geom("48x36x30")
    cats = _columns(C, radius, 34)
    e = np.linspace(0, rmax, 5)
    a = _run(cats, N, L, C, cplx, "tsc", True, edges=e)
    b = _run(cats, N, L, C, real, "tsc", True, edges=e)
    Nf, Rf = _fields(b)
    want = cfo.fft_form(Nf, Rf, N, L, e, POLES)
    np.testing.assert_array_equal(a.nsep, b.nsep)
    # the same paint; f4 paints differ in the order of their float32 atomic adds
    tol = 1e-12 if real == "f8" else 1e-6
    for kind, bk in (("nnn", "bound_n"), ("rrr", "bound_r")):
        err = np.abs(_stack(a, kind) - _stack(b, kind)) / want[bk]
        assert err.max() <= tol, (kind, err.max())


@pytest.mark.parametrize("cap", [3, 4])
def test_blocked_path_matches_resident(cuda, monkeypatch, cap):
    from nbodykit_b200.algorithms.fft3pcf import bin_blocks, transform_count
    N, L, C, rmax, radius = _geom("32")
    cats = _columns(C, radius, 35)
    e = np.linspace(0, rmax, 7)
    one = _run(cats, N, L, C, "f8", "cic", edges=e)
    monkeypatch.setenv("NBK_BISPEC_RESIDENT", str(cap))
    blk = _run(cats, N, L, C, "f8", "cic", edges=e)
    assert blk.attrs["transforms"] == transform_count(bin_blocks(6, cap), POLES, 2) > one.attrs["transforms"]
    Nf, Rf = _fields(one)
    want = cfo.fft_form(Nf, Rf, N, L, e, POLES)
    for kind, bk in (("nnn", "bound_n"), ("rrr", "bound_r")):
        err = np.abs(_stack(blk, kind) - _stack(one, kind)) / want[bk]
        assert err.max() <= 1e-12, (cap, kind, err.max())
    np.testing.assert_array_equal(blk.nsep, one.nsep)


def _on_ranks(comm, shape, cats, owner):
    N, L, C, rmax, _ = _geom(shape)
    r = _run(cats, N, L, C, "f8", "tsc", True, comm=comm, owner=owner, edges=np.linspace(0, rmax, 5))
    return dict(nnn=_stack(r, "nnn"), rrr=_stack(r, "rrr"), nsep=r.nsep, transforms=r.attrs["transforms"],
                tiles=r.attrs["tiles"])


@pytest.mark.parametrize("shape,P", [("32", 2), ("48x36x30", 3), ("32", 4)])
def test_ranks_match_one(cuda, shape, P):
    from test_gpu_slab_route import _spawn
    N, L, C, rmax, radius = _geom(shape)
    cats = _columns(C, radius, 37)
    rng = np.random.RandomState(3)
    owner = {name: rng.randint(0, P, len(c["NZ"])) for name, c in cats.items()}
    e = np.linspace(0, rmax, 5)
    one = _run(cats, N, L, C, "f8", "tsc", True, edges=e)
    Nf, Rf = _fields(one)
    want = cfo.fft_form(Nf, Rf, N, L, e, POLES)
    parts = _spawn(_on_ranks, P, shape, cats, owner)
    for rank, part in enumerate(parts):
        np.testing.assert_array_equal(part["nsep"], one.nsep)
        for kind, bk in (("nnn", "bound_n"), ("rrr", "bound_r")):
            err = np.abs(part[kind] - _stack(one, kind)) / want[bk]
            assert err.max() <= 1e-12, (shape, rank, kind, err.max())
        assert part["transforms"] == one.attrs["transforms"]
        assert 0 < part["tiles"] <= 1


def test_two_gpu_convfft3pcf_matches_one_gpu():
    """launches tests/mgpu_check_convfft3pcf.py under torchrun when the box has >= 2 GPUs"""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29553", os.path.join(ROOT, "tests", "mgpu_check_convfft3pcf.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    sys.stdout.write(out.stdout[-3000:])
    sys.stderr.write(out.stderr[-3000:])
    assert out.returncode == 0
