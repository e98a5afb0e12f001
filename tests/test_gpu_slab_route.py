"""
Particle routing (csrc/route.cu) into the slab paint and the slab readout on P virtual ranks of one GPU, against
float64 NumPy (oracle/pmesh_oracle.py, recon_oracle.py, mesh_layouts.py).

Every virtual rank holds its own local catalogue, routes it with nbk_route_count + nbk_route_scatter and receives
segment r of every rank's send buffer, in rank order (SlabLayout.route).  The routing contract is checked against the
paint stencil itself: every rank that owns a plane a particle deposits on is its own rank or in its routed mask.
Each rank then paints its local particles (clear) and the received ones (hold) into its x slab, and the joined slabs
must equal the one-mesh paint; the readout partial sums of the local and received rows, added back over send_index
(RealField.readout's gather_back), must equal the one-mesh readout.

The last test runs the same glue through pm.py itself: P = 2 and 4 processes over gloo (127.0.0.1) share device 0 with
the all-to-all transpose (NBK_FFT_TRANSPOSE=nccl), and compensated paints (the P > 1 c2r), the interlaced PCS routing,
a shifted readout and FFTRecon must equal one process.
"""
import datetime
import os
import socket
import sys

import numpy as np
import pytest
from gpu_helpers import code as _code, dev as _dev, host as _host, nbk as _lib, ptr as _p

from oracle import mesh_layouts as ml
from oracle import pmesh_oracle as po
from oracle import recon_oracle as ro

pytestmark = pytest.mark.gpu

WINDOWS = ["nnb", "cic", "tsc", "pcs"]
# (N, P): x_n = 16; x_n = 5 (the thinnest tiled PCS slab, x_start off the 16-cell tiles); x_n = 4 (interlaced PCS reaches
# three slabs: the loop branch of route_mask); x_n = 16 at P = 4; x_n = 2 at the route's 32 ranks (direct paint only)
GEOMS = {"48x32x32-P3": ((48, 32, 32), 3), "40x32x32-P8": ((40, 32, 32), 8), "32x32x32-P8": ((32, 32, 32), 8),
         "64x32x32-P4": ((64, 32, 32), 4), "64x16x16-P32": ((64, 16, 16), 32)}
# N / L a power of two on every axis (the paint's float32 shortcut) or not
BOXES = {"pow2": lambda N: tuple(0.5 * n for n in N), "margin": lambda N: (100., 3.3, 7000.)}
# (position dtype, mass dtype or None)
COLUMNS = [("f4", None), ("f8", "f4"), ("f4", "f8")]
SPLITS = ["random", "slab-local", "all-remote"]


def paint_smoothing(res, interlaced):
    """what source/mesh/catalog.py passes to decompose"""
    return (1.0 if interlaced else 0.5) * po.SUPPORT[res]


def readout_smoothing(res, shift):
    """what RealField.readout passes to decompose"""
    return 0.5 * po.SUPPORT[res] + abs(shift)


def _owner(pos, N, L, P, split, seed):
    """the rank holding each particle"""
    Nx = N[0]
    slab = (np.floor(pos[:, 0].astype("f8") * (Nx / L[0])).astype("i8") % Nx) // (Nx // P)
    if split == "slab-local":
        return slab
    if split == "all-remote":
        return (slab - 1) % P                 # rank r holds the particles of slab r + 1
    return np.random.RandomState(seed).randint(0, P, size=len(pos))


class Rank(object):
    """one virtual rank: its local catalogue (host + device) and, after route(), what it sent"""

    def __init__(self, pos, mass):
        self.pos, self.mass = pos, mass
        self.dpos = _dev(pos)
        self.dmass = None if mass is None else _dev(mass)


def route(ranks, N, L, P, s):
    """nbk_route_count + nbk_route_scatter on every rank; returns per rank (mask per local row, counts, send pos, send
    mass, send index) and checks the list and segment invariants"""
    import torch
    _l = _lib()
    sent = []
    for r, rk in enumerate(ranks):
        n = len(rk.pos)
        counts = torch.zeros(P + 1, dtype=torch.int64, device="cuda")
        lst = torch.empty(max(n, 1), dtype=torch.int64, device="cuda")
        _l.check(_l.lib().nbk_route_count(_p(rk.dpos), _code(rk.pos.dtype), n, s, _l.darr(L), _l.iarr(N), P, r,
                                          _p(counts), _p(lst), None), "nbk_route_count")
        c = _host(counts)
        nl = int(c[P])
        ent = _host(lst)[:nl].view(np.uint64)
        idx, mask = (ent & np.uint64(0xffffffff)).astype("i8"), (ent >> np.uint64(32)).astype("i8")
        assert len(np.unique(idx)) == nl, "a particle listed twice"
        assert (mask != 0).all() and not ((mask >> r) & 1).any(), "empty or own-rank destination"
        cnt = [int(((mask >> q) & 1).sum()) for q in range(P)]
        assert c[:P].tolist() == cnt
        full = np.zeros(n, dtype="i8")
        full[idx] = mask
        tot = sum(cnt)
        off = torch.tensor([0] + list(np.cumsum(cnt)[:-1]), dtype=torch.int64, device="cuda")
        cur = torch.zeros(P, dtype=torch.int64, device="cuda")
        spos = torch.empty((tot, 3), dtype=rk.dpos.dtype, device="cuda")
        smass = None if rk.mass is None else torch.empty(tot, dtype=rk.dmass.dtype, device="cuda")
        sidx = torch.empty(tot, dtype=torch.int64, device="cuda")
        _l.check(_l.lib().nbk_route_scatter(_p(rk.dpos), _code(rk.pos.dtype), _p(rk.dmass),
                                            _code(rk.mass.dtype) if rk.mass is not None else 8, _p(lst), nl, P, _p(off),
                                            _p(cur), _p(spos), _p(smass), _p(sidx), None), "nbk_route_scatter")
        si = _host(sidx)
        assert np.array_equal(_host(spos), rk.pos[si]), "sidx does not point at the rows copied"
        if rk.mass is not None:
            assert np.array_equal(_host(smass), rk.mass[si])
        b = 0
        for q in range(P):
            seg = si[b:b + cnt[q]]
            assert np.array_equal(np.sort(seg), np.flatnonzero((full >> q) & 1)), "segment %d of rank %d" % (q, r)
            b += cnt[q]
        sent.append(dict(mask=full, counts=cnt, spos=spos, smass=smass, sidx=sidx))
    return sent


def received(sent, r):
    """what rank r receives: segment r of every rank q, in rank order (positions, masses, per source rank (q, rows))"""
    import torch
    parts, masses, rows = [], [], []
    for q, sq in enumerate(sent):
        a = sum(sq["counts"][:r])
        b = a + sq["counts"][r]
        parts.append(sq["spos"][a:b])
        if sq["smass"] is not None:
            masses.append(sq["smass"][a:b])
        rows.append((q, a, b))
    pos = torch.cat(parts).contiguous()
    mass = torch.cat(masses).contiguous() if masses else None
    return pos, mass, rows


def check_contract(ranks, sent, N, L, P, res, shifts, what):
    """every rank owning a plane of a particle's stencil is its own rank or in its routed mask"""
    for r, (rk, sr) in enumerate(zip(ranks, sent)):
        need = ml.stencil_ranks(rk.pos, N, L, P, res, shifts) & ~(1 << r)
        miss = need & ~sr["mask"]
        if miss.any():
            i = int(np.flatnonzero(miss)[0])
            raise AssertionError("%s: rank %d, particle x = %r (g = %.17g) deposits on ranks %s but is routed to %s"
                                 % (what, r, rk.pos[i, 0], rk.pos[i, 0].astype("f8") * N[0] / L[0], bin(need[i]),
                                    bin(sr["mask"][i])))


def _catalogue(geom, box, pdt, mdt):
    """uniform particles under slab-edge ones for every smoothing the call sites pass"""
    N, P = GEOMS[geom]
    L = BOXES[box](N)
    smooth = sorted({paint_smoothing(w, i) for w in WINDOWS for i in (False, True)} |
                    {readout_smoothing(w, s) for w in WINDOWS for s in (0.0, 0.5)})
    pos, _ = ml.slab_edge_positions(N, L, P, smooth, pdt, n_uniform=6000, seed=len(geom))
    rng = np.random.RandomState(3)
    mass = None if mdt is None else rng.uniform(0.1, 3.0, size=len(pos)).astype(mdt)
    return N, P, L, pos, mass


def _ranks(pos, mass, N, L, P, split):
    own = _owner(pos, N, L, P, split, 5)
    return own, [Rank(pos[own == r], None if mass is None else mass[own == r]) for r in range(P)]


def _slab_paint(kind, N, L, P, r, batches, res, x_n, shift=0.0):
    """one rank: paint the batches (local first, clear; then received, hold) into its slab(s) with path `kind`"""
    import torch
    _l = _lib()
    Lb = _l.lib()
    m1 = torch.zeros((x_n, N[1], N[2]), dtype=torch.float64, device="cuda")
    m2 = torch.zeros_like(m1) if kind in ("interlaced", "tiled-pair") else None
    w = _l.WINDOW[res]
    first = True
    for p, m in batches:
        n = int(p.shape[0])
        if n == 0:
            continue
        pc = 4 if p.dtype == torch.float32 else 8
        mc = (4 if m.dtype == torch.float32 else 8) if m is not None else 8
        args = (_l.darr(L), _l.iarr(N), r * x_n, x_n)
        if kind == "direct":
            _l.check(Lb.nbk_paint(_p(p), pc, n, _p(m), mc, w, 0.0, *args, _p(m1), 8, None), "nbk_paint")
        elif kind == "interlaced":
            _l.check(Lb.nbk_paint_interlaced(_p(p), pc, n, _p(m), mc, w, *args, _p(m1), _p(m2), 8, None),
                     "nbk_paint_interlaced")
        else:
            nb = int(Lb.nbk_paint_tiled_workspace(n, pc, mc if m is not None else 0, _l.iarr(N), x_n))
            work = torch.empty(max(nb, 1), dtype=torch.uint8, device="cuda")
            _l.check(Lb.nbk_paint_tiled(_p(p), pc, n, _p(m), mc, w, shift, *args, _p(m1), _p(m2), 8, _p(work), nb,
                                        1 if first else 0, None), "nbk_paint_tiled")
        first = False
    return [_host(m1)] + ([_host(m2)] if m2 is not None else [])


# ---------------------------------------------------------------------------------------------
# routing + paint
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geom", sorted(GEOMS))
@pytest.mark.parametrize("box", sorted(BOXES))
@pytest.mark.parametrize("cols", COLUMNS, ids=lambda c: "pos%s-mass%s" % c)
def test_route_then_paint_equals_one_mesh(cuda, geom, box, cols):
    """three catalogue splits x four windows: the routing contract for the smoothing of the plain and the interlaced
    paint, then direct, interlaced, tiled and tiled-pair paint of local + received particles on every slab against the
    one-mesh po.paint; tiled NNB bit for bit against the per-batch fixed-point sums; mass conserved"""
    _l = _lib()
    N, P, L, pos, mass = _catalogue(geom, box, cols[0], cols[1])
    x_n = N[0] // P
    total = len(pos) if mass is None else float(mass.astype("f8").sum())
    want = {(res, s): po.paint(pos, mass, N, L, res, s) for res in WINDOWS for s in (0.0, 0.5)}
    # every cell of slab r gets the deposits of the whole catalogue in that cell, in two batches whose fixed-point
    # scales are at most that of the whole catalogue: the one-batch bound of the whole catalogue holds
    bound = {(res, s): ml.deposit_bound(pos, mass, N, L, res, s)[0] for res in WINDOWS for s in (0.0, 0.5)}
    for split in SPLITS:
        _, ranks = _ranks(pos, mass, N, L, P, split)
        for res in WINDOWS:
            tiled = bool(_l.lib().nbk_paint_tiled_supported(_l.iarr(N), x_n, _l.WINDOW[res]))
            for interlaced in (False, True):
                s = paint_smoothing(res, interlaced)
                shifts = (0.0, 0.5) if interlaced else (0.0,)
                what = "%s %s %s s=%g" % (split, res, "interlaced" if interlaced else "plain", s)
                sent = route(ranks, N, L, P, s)
                check_contract(ranks, sent, N, L, P, res, shifts, what)
                kinds = (["interlaced"] + (["tiled-pair"] if tiled else [])) if interlaced else \
                    (["direct"] + (["tiled"] if tiled else []))
                recv = [received(sent, r) for r in range(P)]
                for kind in kinds:
                    slabs = [_slab_paint(kind, N, L, P, r, [(rk.dpos, rk.dmass), recv[r][:2]], res, x_n)
                             for r, rk in enumerate(ranks)]
                    for j, shift in enumerate(shifts):
                        got = np.concatenate([sl[j] for sl in slabs])
                        w, bd = want[res, shift], bound[res, shift]
                        tag = "%s %s shift %g" % (what, kind, shift)
                        np.testing.assert_allclose(got.sum(), total, rtol=1e-9, err_msg=tag + ": mass")
                        if kind.startswith("tiled"):
                            err = np.abs(got - w)
                            assert (err <= bd).all(), "%s: worst %g > bound" % (tag, (err - bd).max())
                            if res == "nnb":
                                exact = []
                                for r, rk in enumerate(ranks):
                                    rp, rm = _host(recv[r][0]), (None if recv[r][1] is None else _host(recv[r][1]))
                                    e = ml.nnb_fixed_point(rk.pos, rk.mass, N, L, shift) + \
                                        ml.nnb_fixed_point(rp, rm, N, L, shift)
                                    exact.append(e[r * x_n:(r + 1) * x_n])
                                assert np.array_equal(got, np.concatenate(exact)), tag + ": NNB not bit-exact"
                        else:
                            np.testing.assert_allclose(got, w, rtol=0, atol=1e-12 * np.abs(w).max(), err_msg=tag)


@pytest.mark.parametrize("res", WINDOWS)
@pytest.mark.parametrize("box", sorted(BOXES))
def test_tiled_shifted_mesh_follows_rounding_contract(cuda, res, box):
    """one mesh (P = 1), f8 positions and f4 masses: the half-cell shifted mesh of the tiled paint -- the second mesh of
    the interlaced pair and a single mesh at shift 1/2 -- within the per-cell deposit bound of the contract g' =
    fl(g + 1/2).  The catalogue holds g = k + 1/2 - 2^-j (j = 1 .. 3 ulp): g + 1/2 rounds up onto the integer k + 1 in
    f8, so the shifted stencil starts at k + 1; the fixed-point carry of frac(g) + 1/2 alone started it at k and left a
    2^-28 weight on cell k (seen first at x = 1/2 - 2^-54 cells on a 64^3-slab catalogue)."""
    N, P, L, pos, mass = _catalogue("64x32x32-P4", box, "f8", "f4")
    Nx = N[0]
    # g = k + 1/2 - ulps for cells across the mesh, the seam and an image one box length out
    near = []
    for k in (0, 1, 7, Nx // 2, Nx - 1, Nx, -1, Nx + 3):
        for v in ml._ulp_neighbours((k + 0.5) * L[0] / Nx, "f8"):
            near.append(float(v))
    extra = np.random.RandomState(4).uniform(0, 1, size=(len(near), 3)) * np.asarray(L)
    extra[:, 0] = near
    pos = np.concatenate([pos, extra])
    mass = np.concatenate([mass, np.full(len(near), 0.5, dtype=mass.dtype)])
    _, ranks = _ranks(pos, mass, N, L, 1, "random")
    rk = ranks[0]
    want = {s: po.paint(pos, mass, N, L, res, s) for s in (0.0, 0.5)}
    bound = {s: ml.deposit_bound(pos, mass, N, L, res, s)[0] for s in (0.0, 0.5)}
    pair = _slab_paint("tiled-pair", N, L, 1, 0, [(rk.dpos, rk.dmass)], res, Nx)
    single = _slab_paint("tiled", N, L, 1, 0, [(rk.dpos, rk.dmass)], res, Nx, shift=0.5)[0]
    for got, shift, what in ((pair[0], 0.0, "pair, mesh 1"), (pair[1], 0.5, "pair, shifted mesh"),
                             (single, 0.5, "single shifted mesh")):
        err = np.abs(got - want[shift])
        assert (err <= bound[shift]).all(), "%s: worst %g > bound" % (what, (err - bound[shift]).max())


# ---------------------------------------------------------------------------------------------
# routing + readout + gather back
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geom", sorted(GEOMS))
@pytest.mark.parametrize("box", sorted(BOXES))
@pytest.mark.parametrize("pdt", ["f4", "f8"])
def test_route_readout_gather_back_equals_one_mesh(cuda, geom, box, pdt):
    """per rank: readout of the local rows into an f8 accumulator, readout of the received rows, their partial sums
    added back over send_index -- equal to ro.readout on the whole mesh, four windows, shifts 0 and 0.5, f8 and f4
    meshes, three catalogue splits"""
    import torch
    _l = _lib()
    N, P, L, pos, _ = _catalogue(geom, box, pdt, None)
    x_n = N[0] // P
    field8 = np.random.RandomState(17).standard_normal(N)
    fields = {"f8": field8, "f4": field8.astype("f4")}
    slabs = {m: [_dev(f[r * x_n:(r + 1) * x_n]) for r in range(P)] for m, f in fields.items()}
    want = {(m, res, sh): ro.readout(f.astype("f8"), pos, N, L, res, sh) for m, f in fields.items() for res in WINDOWS
            for sh in (0.0, 0.5)}

    def rd(mdt, r, p, out, res, shift):
        if p.shape[0]:
            _l.check(_l.lib().nbk_readout(_p(slabs[mdt][r]), _code(mdt), _p(p), _code(pdt), int(p.shape[0]),
                                          _l.WINDOW[res], shift, _l.darr(L), _l.iarr(N), r * x_n, x_n, _p(out), 8, 0,
                                          None), "nbk_readout")
    for split in SPLITS:
        own, ranks = _ranks(pos, None, N, L, P, split)
        for res in WINDOWS:
            for shift in (0.0, 0.5):
                s = readout_smoothing(res, shift)
                what = "%s %s shift %g s=%g" % (split, res, shift, s)
                sent = route(ranks, N, L, P, s)
                check_contract(ranks, sent, N, L, P, res, (shift,), what)
                recv = [received(sent, r) for r in range(P)]
                for mdt in ("f8", "f4"):
                    accs = []
                    for r, rk in enumerate(ranks):
                        acc = torch.empty(len(rk.pos), dtype=torch.float64, device="cuda")
                        rd(mdt, r, rk.dpos, acc, res, shift)
                        accs.append(acc)
                    for r in range(P):
                        rpos, _, rows = recv[r]
                        part = torch.empty(int(rpos.shape[0]), dtype=torch.float64, device="cuda")
                        rd(mdt, r, rpos, part, res, shift)
                        k = 0
                        for q, a, b in rows:           # the rows rank q sent to r travel back and are added
                            accs[q].index_add_(0, sent[q]["sidx"][a:b], part[k:k + b - a])
                            k += b - a
                    got = np.empty(len(pos))
                    for r in range(P):
                        got[own == r] = _host(accs[r])
                    w = want[mdt, res, shift]
                    tol = (1e-12 if mdt == "f8" else 1e-6) * np.abs(w).max()
                    np.testing.assert_allclose(got, w, rtol=0, atol=tol, err_msg="%s mesh %s" % (what, mdt))


# ---------------------------------------------------------------------------------------------
# end to end through pm.py on gloo ranks sharing device 0
# ---------------------------------------------------------------------------------------------
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E2E_N, E2E_L = 32, 200.


def _free_port():
    sk = socket.socket()
    sk.bind(("127.0.0.1", 0))
    port = sk.getsockname()[1]
    sk.close()
    return port


def _worker(rank, world, port, fn, args, ret):
    import torch
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["NBK_FFT_TRANSPOSE"] = "nccl"
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
    try:
        from nbodykit_b200.comm import TorchComm
        ret[rank] = fn(TorchComm(), *args)
    finally:
        dist.destroy_process_group()


def _spawn(fn, world, *args):
    """runs fn(comm, *args) on `world` processes sharing device 0; every process is joined before this returns"""
    import torch.multiprocessing as mp
    mgr = mp.Manager()
    try:
        ret = mgr.dict()
        mp.spawn(_worker, args=(world, _free_port(), fn, args, ret), nprocs=world, join=True)
        return [ret[r] for r in range(world)]
    finally:
        mgr.shutdown()


def _e2e(comm, data, ran):
    """this rank's share of: two compensated paints taken back to real space, a shifted CIC readout of the first
    at this rank's particles, FFTRecon (LGS), each as numpy (real fields: this rank's x slab)"""
    import torch
    from nbodykit_b200.lab import ArrayCatalog, FFTRecon

    def mine(a):
        return a[comm.rank * len(a) // comm.size:(comm.rank + 1) * len(a) // comm.size]

    def cat(a):
        return ArrayCatalog({"Position": torch.from_numpy(mine(a)).cuda()}, comm=comm, BoxSize=E2E_L, Nmesh=E2E_N)
    d = cat(data)
    out = {}
    tsc = d.to_mesh(resampler="tsc", compensated=True, dtype="f8").compute(mode="real")
    out["tsc"] = tsc.numpy()
    out["pcs-interlaced"] = d.to_mesh(resampler="pcs", interlaced=True, compensated=True,
                                      dtype="f8").compute(mode="real").numpy()
    pm = tsc.pm
    out["readout"] = tsc.readout(mine(data), resampler="cic", transform=pm.affine.shift(0.5))
    rec = FFTRecon(data=d, ran=cat(ran), Nmesh=E2E_N, bias=1.5, f=0.0, los=[0, 0, 1], R=20., scheme="LGS")
    out["recon"] = rec.compute(mode="real").numpy()
    return out


@pytest.mark.parametrize("P", [2, 4])
def test_pm_slab_glue_on_ranks_equals_one(cuda, P):
    """the smoothing of each call site, SlabLayout.route / gather_back and the P > 1 c2r, through pm.py: at P = 4 the
    32-plane mesh has x_n = 8, which interlaced PCS (a 9-cell reach) overruns"""
    from nbodykit_b200.comm import SelfComm
    rng = np.random.RandomState(41)
    data = (rng.uniform(0, 1, size=(30000, 3)) * E2E_L).astype("f4")
    data[:2000, 0] = (rng.randint(0, E2E_N, size=2000) + rng.choice([-1e-4, 0.5, 1e-4], size=2000)) * (E2E_L / E2E_N)
    ran = (rng.uniform(0, 1, size=(60000, 3)) * E2E_L).astype("f4")
    one = _e2e(SelfComm(), data, ran)
    parts = _spawn(_e2e, P, data, ran)
    for key in ("tsc", "pcs-interlaced", "readout", "recon"):
        got = np.concatenate([p[key] for p in parts])
        want = one[key]
        assert got.shape == want.shape, key
        # the recon fields shift float32 positions by displacements whose last bits depend on the summation order
        tol = (1e-5 if key == "recon" else 1e-12) * np.abs(want).max()
        np.testing.assert_allclose(got, want, rtol=0, atol=tol, err_msg="%s P=%d" % (key, P))
