"""
The mesh-stage kernels on the layouts every P > 1 run uses, at odd and Nyquist-carrying mesh sides, against float64
NumPy references (oracle/pmesh_oracle.py, recon_oracle.py, convpower_oracle.py, mesh_layouts.py).

P virtual ranks run on one GPU: rank r gets its slab as its own contiguous array and is called with the layout bits,
start and count that pm.py passes (transposed y slabs [y_n][Nx][Nzc] in Fourier space, x slabs [x_n][Ny][Nz] in real
space); the slabs are reassembled (or the per-rank accumulators summed) and compared with the full-mesh reference.
The tiled paint is driven with particles on and around the cell boundaries of its index arithmetic, and its
fixed-point scale is pinned bit for bit.
"""
import ctypes

import numpy as np
import pytest

from oracle import convpower_oracle as co
from oracle import mesh_layouts as ml
from oracle import pmesh_oracle as po
from oracle import recon_oracle as ro

pytestmark = pytest.mark.gpu

SIDES = [(45, 21, 35), (44, 52, 37), (48, 36, 17), (30, 33, 16), (32, 32, 32)]
BOX = (100., 130., 70.)
LAYOUT_TRANSPOSED, LAYOUT_FULLZ = 1, 2
COMP_NAMES = ["CompensateCIC", "CompensateTSC", "CompensatePCS", "CompensateCICShotnoise", "CompensateTSCShotnoise",
              "CompensatePCSShotnoise"]


def _lib():
    from nbodykit_b200 import _lib
    return _lib


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _code(dtype):
    return 4 if dtype == "f4" else 8


def _host(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy()


def _layouts(N):
    """0: the untransposed whole mesh (P = 1); P >= 1: P transposed y slabs (P = 1 is the whole mesh transposed)"""
    return [0, 1] + ml.rank_counts(N[1])


def _on_slabs(arrays, N, P, fn):
    """run fn(device tensors, layout, start, count) on every virtual rank of layout P (see _layouts) and return the
    reassembled arrays"""
    if P == 0:
        ts = [_dev(a) for a in arrays]
        fn(ts, 0, 0, N[0])
        return [_host(t) for t in ts]
    y_n = N[1] // P
    per_rank = []
    for r, parts in enumerate(zip(*[ml.split_transposed(a, P) for a in arrays])):
        ts = [_dev(a) for a in parts]
        fn(ts, LAYOUT_TRANSPOSED, r * y_n, y_n)
        per_rank.append([_host(t) for t in ts])
    return [ml.join_transposed([pr[i] for pr in per_rank]) for i in range(len(arrays))]


def _close(got, want, tol):
    err = np.abs(got - want).max()
    assert err <= tol * np.abs(want).max(), "max error %g > %g x max |want| %g" % (err, tol, np.abs(want).max())


# ---------------------------------------------------------------------------------------------
# A. element-wise Fourier-space kernels
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", SIDES)
@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_compensate_layouts(cuda, N, dtype):
    """all six transfer functions, every virtual-rank split of the transposed slabs, and the full-z layout"""
    _l = _lib()
    c, full = ml.spectra(N, np.random.RandomState(1), dtype)
    tol = 1e-13 if dtype == "f8" else 2e-7
    for name in COMP_NAMES:
        kind = _l.COMP[name]
        want = po.compensate(name, ml.k_coords(N, BOX, "f8", kind="circular"), c.astype("c16"))

        def run(ts, lay, start, count):
            _l.check(_l.lib().nbk_compensate(_ptr(ts[0]), _code(dtype), kind, _l.iarr(N), lay, start, count, None))
        for P in _layouts(N):
            got, = _on_slabs([c], N, P, run)
            np.testing.assert_allclose(got, want, rtol=tol, atol=0, err_msg="%s P=%d" % (name, P))
        t = _dev(full)
        _l.check(_l.lib().nbk_compensate(_ptr(t), _code(dtype), kind, _l.iarr(N), LAYOUT_FULLZ, 0, N[0], None))
        wantf = po.compensate(name, ml.k_coords(N, BOX, "f8", kind="circular", fullz=True), full.astype("c16"))
        np.testing.assert_allclose(_host(t), wantf, rtol=tol, atol=0, err_msg="%s full z" % name)


@pytest.mark.parametrize("N", SIDES)
@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_interlace_combine_layouts(cuda, N, dtype):
    _l = _lib()
    rng = np.random.RandomState(2)
    c1, f1 = ml.spectra(N, rng, dtype)
    c2, f2 = ml.spectra(N, rng, dtype)
    tol = 1e-13 if dtype == "f8" else 2e-6
    want = po.interlace_combine(c1.astype("c16"), c2.astype("c16"), N, BOX, "f8")
    np.testing.assert_allclose(ml.interlace_ref(c1.astype("c16"), c2.astype("c16"), N, BOX), want, rtol=1e-14)

    def run(ts, lay, start, count):
        _l.check(_l.lib().nbk_interlace_combine(_ptr(ts[0]), _ptr(ts[1]), _code(dtype), _l.iarr(N), _l.darr(BOX), lay,
                                                start, count, None))
    for P in _layouts(N):
        got, _ = _on_slabs([c1, c2], N, P, run)
        _close(got, want, tol)
    t1, t2 = _dev(f1), _dev(f2)
    run([t1, t2], LAYOUT_FULLZ, 0, N[0])
    _close(_host(t1), ml.interlace_ref(f1.astype("c16"), f2.astype("c16"), N, BOX, fullz=True), tol)


@pytest.mark.parametrize("N", SIDES)
@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_recon_displacement_layouts(cuda, N, dtype):
    """three axes, oblique line of sight"""
    _l = _lib()
    c, full = ml.spectra(N, np.random.RandomState(3), dtype)
    R, bias, f, los = 15., 2.0, 0.7, (0.6, 0., 0.8)
    tol = 1e-13 if dtype == "f8" else 2e-6
    for axis in range(3):
        want = ro.displacement_modes(c.astype("c16"), N, BOX, axis, R, bias, f, los)

        def run(ts, lay, start, count):
            _l.check(_l.lib().nbk_recon_displacement(_ptr(ts[0]), _ptr(ts[1]), _code(dtype), _l.iarr(N), _l.darr(BOX),
                                                     lay, start, count, axis, R, bias, f, _l.darr(los), None))
        for P in _layouts(N):
            _, got = _on_slabs([c, np.zeros_like(c)], N, P, run)
            _close(got, want, tol)
        ts = [_dev(full), _dev(np.zeros_like(full))]
        run(ts, LAYOUT_FULLZ, 0, N[0])
        _close(_host(ts[1]), ml.recon_ref(full.astype("c16"), N, BOX, axis, R, bias, f, los, fullz=True), tol)


# ---------------------------------------------------------------------------------------------
# B. binning: raw accumulators per virtual rank
# ---------------------------------------------------------------------------------------------
def _edges(N, Nmu):
    Lv = np.asarray(BOX)
    dk = 2 * np.pi / Lv.min()
    return np.arange(0., np.pi * min(N) / Lv.max() + dk / 2, dk), np.linspace(-1, 1, Nmu + 1)


def _bin(fields, N, dtype, lay, start, count, edges, los, ells, herm, coord, is_p3d=False, V=1.0, clear=True,
         comp=(None, None)):
    """one nbk_power_bin / nbk_power_bin2 call (fields: c1 [, c2 [, c2_mirror]] device tensors) -> host raw sums
    (nsum, xsum, musum, ysum[Nell][nb] complex)"""
    import torch
    _l = _lib()
    kedges, muedges = edges
    Nx, Nmu = len(kedges) - 1, len(muedges) - 1
    nb = (Nx + 2) * (Nmu + 2)
    nsum = torch.zeros(nb, dtype=torch.int64, device="cuda")
    xsum = torch.zeros(nb, dtype=torch.float64, device="cuda")
    musum = torch.zeros(nb, dtype=torch.float64, device="cuda")
    ysum = torch.zeros(len(ells) * nb * 2, dtype=torch.float64, device="cuda")
    c1, c2, c3 = (list(fields) + [None, None])[:3]
    fn = _l.lib().nbk_power_bin if c3 is None else _l.lib().nbk_power_bin2
    extra = () if c3 is None else (_ptr(c3),)
    _l.check(fn(_ptr(c1), _ptr(c2), *extra, _code(dtype), 1 if is_p3d else 0, float(V), 1 if clear else 0, _l.iarr(N),
                _l.darr(BOX), lay, start, count, coord, _l.darr(np.asarray(kedges) ** 2), Nx, _l.darr(muedges), Nmu,
                _l.darr(los), _l.i32arr(ells), len(ells), herm, _l.COMP.get(comp[0], 0), _l.COMP.get(comp[1], 0), 0, None,
                _ptr(nsum), _ptr(xsum), _ptr(musum), _ptr(ysum), None), "nbk_power_bin")
    y = _host(ysum).reshape(len(ells), nb, 2)
    return _host(nsum), _host(xsum), _host(musum), y[..., 0] + 1j * y[..., 1]


def _bin_layout(arrays, N, P, dtype, **kw):
    """the raw sums of layout P (see _layouts), summed over the virtual ranks"""
    if P == 0:
        return _bin([_dev(a) for a in arrays], N, dtype, 0, 0, N[0], **kw)
    y_n = N[1] // P
    tot = None
    for r, parts in enumerate(zip(*[ml.split_transposed(a, P) for a in arrays])):
        s = _bin([_dev(a) for a in parts], N, dtype, LAYOUT_TRANSPOSED, r * y_n, y_n, **kw)
        tot = s if tot is None else tuple(a + b for a, b in zip(tot, s))
    return tot


def _check_sums(got, want, tol, what, mu=True):
    """counts bit-exact; x, mu, y sums within tol relative (and tol x max |want| absolute)"""
    ng, xg, mg, yg = got
    nw, xw, mw, yw = [np.asarray(w).reshape(np.shape(g)) for w, g in zip(want, got)]
    assert np.array_equal(ng, nw), "%s: mode counts differ" % what
    pairs = [(xg, xw), (yg, yw)] + ([(mg, mw)] if mu else [])
    for g, w in pairs:
        np.testing.assert_allclose(g, w, rtol=tol, atol=tol * max(np.abs(w).max(), 1e-300), err_msg=what)


def _stat(c1, c2, N, kind, V, clear, comp):
    """the 3-D statistic the kernel forms on the fly, in f8"""
    if kind == "p3d":
        return c1.astype("c16")
    a, b = c1.astype("c16"), (c1 if c2 is None else c2).astype("c16")
    w = ml.k_coords(N, BOX, "f8", kind="circular")
    if comp[0]:
        a = po.compensate(comp[0], w, a)
        b = po.compensate(comp[1] if c2 is not None else comp[0], w, b)
    y = a * np.conj(b)
    if clear:
        y[0, 0, 0] = 0
    return y * V


# id: (N, dtype, los, coord mode, statistic, compensation pair, Nmu, poles, hermitian, clear_zero)
# lean-*: the LEAN instance (auto power, f4 coordinates); z line of sight: the SYM mirror-row grouping
BIN_CASES = {
    "lean-z-odd": ((45, 21, 35), "f8", (0., 0., 1.), 4, "auto", (None, None), 1, [], 1, True),
    "lean-z-comp": ((44, 52, 37), "f4", (0., 0., 1.), 4, "auto", ("CompensateTSCShotnoise",) * 2, 5, [0, 2, 4], 1, True),
    "lean-oblique-comp": ((48, 36, 17), "f4", (0.6, 0., 0.8), 4, "auto", ("CompensatePCSShotnoise",) * 2, 4, [0, 2, 4], 1,
                          True),
    "cross-y": ((48, 36, 17), "f8", (0., 1., 0.), 8, "cross", (None, None), 4, [0, 2, 4], 1, True),
    "p3d-oblique-48": ((30, 33, 16), "f8", (0.6, 0., 0.8), 48, "p3d", (None, None), 5, [0, 2, 4], 1, True),
    "cross-comp-z-noclear": ((32, 32, 32), "f8", (0., 0., 1.), 8, "cross", ("CompensateCICShotnoise",
                                                                            "CompensatePCSShotnoise"), 4, [2], 1, False),
    "anti-y-odd": ((45, 21, 35), "f8", (0., 1., 0.), 4, "cross", (None, None), 5, [1, 3], 2, True),
    "anti-z-p3d-48": ((44, 52, 37), "f8", (0., 0., 1.), 48, "p3d", (None, None), 1, [1, 3], 2, True),
    "anti-z-comp-f4": ((30, 33, 16), "f4", (0., 0., 1.), 8, "cross", ("CompensateTSC", "CompensateCIC"), 4, [1, 3], 2, True),
}


def _bin_case(cid, case):
    N, dtype, los, coord, kind, comp, Nmu, poles, herm, clear = case
    rng = np.random.RandomState(31)
    c1, _ = ml.spectra(N, rng, dtype)
    c2 = ml.spectra(N, rng, dtype)[0] if kind == "cross" else None
    V = float(np.prod(BOX))
    ells = [0] + sorted(poles) if 0 not in poles else sorted(poles)
    edges = _edges(N, Nmu)
    y = _stat(c1, c2, N, kind, V, clear, comp)
    if coord == 8:
        x3d, los_o = po.k_coords(N, BOX, "f8"), list(los)
    elif coord == 48:
        x3d, los_o = po.k_coords(N, BOX, "f4"), np.asarray(los, dtype="f8")     # numpy-scalar los: f8 mu
    else:
        x3d, los_o = po.k_coords(N, BOX, "f4"), list(los)
    ref = (ml.project_sums_anti if herm == 2 else po.project_sums)(y, x3d, edges, los_o, poles)
    want = (ref[3], ref[0], ref[1], ref[2])
    arrays = [c1] + ([c2] if c2 is not None else [])
    kw = dict(edges=edges, los=los, ells=ells, herm=herm, coord=coord, is_p3d=(kind == "p3d"), V=V, clear=clear, comp=comp)
    tol = 1e-12 if dtype == "f8" else 2e-6
    one = None
    for P in _layouts(N):
        got = _bin_layout(arrays, N, P, dtype, **kw)
        _check_sums(got, want, tol, "%s P=%d vs project_sums" % (cid, P))
        if one is None:
            one = got
        else:
            _check_sums(got, one, 1e-13, "%s P=%d vs P=1" % (cid, P))


@pytest.mark.parametrize("cid", sorted(BIN_CASES))
def test_power_bin_virtual_ranks(cuda, cid):
    _bin_case(cid, BIN_CASES[cid])


def test_power_bin_edges_global_odd(cuda, monkeypatch):
    """the k edges read from global memory (NBK_BIN_EDGES_GLOBAL) on an odd mesh, all layouts"""
    monkeypatch.setenv("NBK_BIN_EDGES_GLOBAL", "1")
    _bin_case("edges-global-odd", ((45, 21, 35), "f8", (0., 0., 1.), 4, "cross", (None, None), 5, [0, 2], 1, True))


@pytest.mark.parametrize("N", [(45, 21, 35), (44, 52, 37), (48, 36, 16)])
@pytest.mark.parametrize("kind,los,Nmu,poles", [("p3d", (0., 0., 1.), 5, [0, 2, 4]), ("cross", (0.6, 0., 0.8), 4, [0, 1, 2])])
def test_power_bin_fullz_nonhermitian(cuda, N, kind, los, Nmu, poles):
    """the full-z layout with hermitian = 0 (complex-dtype meshes), P = 1, against project_sums over every mode"""
    rng = np.random.RandomState(41)
    _, f1 = ml.spectra(N, rng)
    _, f2 = ml.spectra(N, rng)
    V = float(np.prod(BOX))
    if kind == "p3d":
        y, arrays = f1, [f1]
    else:
        y, arrays = f1 * np.conj(f2) * V, [f1, f2]
        y[0, 0, 0] = 0
    edges = _edges(N, Nmu)
    x3d = ml.k_coords(N, BOX, "f4", fullz=True)
    ref = po.project_sums(y, x3d, edges, list(los), poles, hermitian_symmetric=False)
    got = _bin([_dev(a) for a in arrays], N, "f8", LAYOUT_FULLZ, 0, N[0], edges=edges, los=los, ells=[0] + poles[1:],
               herm=0, coord=4, is_p3d=(kind == "p3d"), V=V)
    _check_sums(got, (ref[3], ref[0], ref[1], ref[2]), 1e-12, "full z")


# ---------------------------------------------------------------------------------------------
# C. the mirror accumulator of ConvolvedFFTPower
# ---------------------------------------------------------------------------------------------
def _ylm(l, m, d):
    return co.real_ylm(l, m, d[0], d[1], d[2])


def _fold_mu1(s):
    """fold the mu == 1 overflow column into the last mu bin (Nmu = 1: the mirror of a mode has the opposite mu)"""
    n, x, mu, y = [np.array(a) for a in s]
    n, x, mu = n.reshape(-1, 3), x.reshape(-1, 3), mu.reshape(-1, 3)
    y = y.reshape(y.shape[0], -1, 3)
    for a in (n, x, mu):
        a[:, 1] += a[:, 2]
        a[:, 2] = 0
    y[..., 1] += y[..., 2]
    y[..., 2] = 0
    return n, x, mu, y


@pytest.mark.parametrize("N", [(32, 32, 32), (48, 36, 16), (44, 52, 37), (45, 21, 35)])
@pytest.mark.parametrize("ell", [1, 2, 3, 5, 8])
def test_mirror_accumulator(cuda, N, ell):
    """A_l = sum_m c_m Y_lm(khat) and its mirror from nbk_ylm_mul_complex_acc2, binned by nbk_power_bin2 on the
    compressed spectrum (P = 1 and transposed virtual ranks), against the full-z hermitian = 0 binning of the completed
    spectrum and a NumPy full-mesh sum; nbk_ylm_mul_complex_acc cell by cell"""
    _l = _lib()
    rng = np.random.RandomState(50 + ell)
    c0, f0 = ml.spectra(N, rng)
    cm, fm = zip(*[ml.spectra(N, rng) for _ in range(2 * ell + 1)])
    khat, mhat = ml.mirror_dirs(N, BOX)
    A_want = sum(cm[i] * _ylm(ell, m, khat) for i, m in enumerate(range(-ell, ell + 1)))
    B_want = sum(cm[i] * _ylm(ell, m, mhat) for i, m in enumerate(range(-ell, ell + 1)))
    kf = ml.k_coords(N, BOX, "f8", fullz=True)
    kn = np.sqrt(sum(k ** 2 for k in kf))
    kn[kn == 0] = np.inf
    A_full = sum(fm[i] * _ylm(ell, m, [k / kn for k in kf]) for i, m in enumerate(range(-ell, ell + 1)))
    V = float(np.prod(BOX))
    edges = _edges(N, 1)
    los, ells = (0., 0., 1.), [0, 2]
    kw = dict(edges=edges, los=los, ells=ells, herm=1, coord=4, V=V)
    one = None
    for P in _layouts(N):
        y_n = N[1] // P if P else 0

        def acc(ts, lay, start, count):
            for i, m in enumerate(range(-ell, ell + 1)):
                ci = ts[3 + i]
                _l.check(_l.lib().nbk_ylm_mul_complex_acc2(_ptr(ts[0]), _ptr(ts[1]), _ptr(ci), 8, ell, m, _l.iarr(N),
                                                           _l.darr(BOX), lay, start, count, None))
                _l.check(_l.lib().nbk_ylm_mul_complex_acc(_ptr(ts[2]), _ptr(ci), 8, ell, m, _l.iarr(N), _l.darr(BOX),
                                                          lay, start, count, None))
        z = np.zeros_like(c0)
        A, B, A1 = _on_slabs([z, z, z] + list(cm), N, P, acc)[:3]
        _close(A, A_want, 1e-13)
        _close(B, B_want, 1e-13)
        _close(A1, A_want, 1e-13)
        # bin A0 conj(A_l) with the mirror field, per rank
        if P == 0:
            got = _bin([_dev(c0), _dev(A), _dev(B)], N, "f8", 0, 0, N[0], **kw)
        else:
            got = None
            for r, parts in enumerate(zip(*[ml.split_transposed(a, P) for a in (c0, A, B)])):
                s = _bin([_dev(a) for a in parts], N, "f8", LAYOUT_TRANSPOSED, r * y_n, y_n, **kw)
                got = s if got is None else tuple(a + b for a, b in zip(got, s))
        got = _fold_mu1(got)
        if one is None:
            one = got
            full = _fold_mu1(_bin([_dev(f0), _dev(A_full)], N, "f8", LAYOUT_FULLZ, 0, N[0], edges=edges, los=los,
                                  ells=ells, herm=0, coord=4, V=V))
            y = f0 * np.conj(A_full) * V
            y[0, 0, 0] = 0
            ref = po.project_sums(y, ml.k_coords(N, BOX, "f4", fullz=True), edges, list(los), [2],
                                  hermitian_symmetric=False)
            ref = _fold_mu1((ref[3], ref[0], ref[1], ref[2]))
            _check_sums(full, ref, 1e-12, "full z vs numpy")
            # the mirror of a mode has the opposite mu: the mu sums of the two layouts differ by construction
            _check_sums(got, full, 1e-12, "compressed + mirror vs full z", mu=False)
        else:
            _check_sums(got, one, 1e-13, "P=%d vs P=1" % P)


# ---------------------------------------------------------------------------------------------
# D. readout and ylm_mul_real on real x slabs
# ---------------------------------------------------------------------------------------------
def _readout_positions(L, n, dtype, seed):
    rng = np.random.RandomState(seed)
    pos = rng.uniform(-0.5, 1.5, size=(n, 3)) * np.asarray(L)      # a quarter outside the box on every side
    pos[:8] = 0.0
    pos[8:16] = np.asarray(L)
    return pos.astype(dtype)


@pytest.mark.parametrize("N,P", [((45, 21, 35), 3), ((48, 36, 17), 2), ((48, 36, 17), 3), ((48, 36, 17), 4),
                                 ((32, 32, 32), 4)])
@pytest.mark.parametrize("pos_dtype", ["f8", "f4"])
def test_readout_x_slabs(cuda, N, P, pos_dtype):
    """per-rank partial sums (x_start, x_n, accumulate = 1) into one output add up to the full-mesh readout"""
    import torch
    _l = _lib()
    rng = np.random.RandomState(61)
    field = rng.standard_normal(N)
    pos = _readout_positions(BOX, 20000, pos_dtype, 62)
    base = rng.standard_normal(len(pos))
    p = _dev(pos)
    pcode = _code(pos_dtype)
    x_n = N[0] // P
    slabs = [_dev(s) for s in ml.split_x(field, P)]
    whole = _dev(field)
    for res in ["nnb", "cic", "tsc", "pcs"]:
        for shift in (0.0, 0.5):
            want = ro.readout(field, pos, N, BOX, res, shift)
            full = torch.empty(len(pos), dtype=torch.float64, device="cuda")
            _l.check(_l.lib().nbk_readout(_ptr(whole), 8, _ptr(p), pcode, len(pos), _l.WINDOW[res], shift, _l.darr(BOX),
                                          _l.iarr(N), 0, N[0], _ptr(full), 8, 0, None))
            out = _dev(base)
            for r in range(P):
                _l.check(_l.lib().nbk_readout(_ptr(slabs[r]), 8, _ptr(p), pcode, len(pos), _l.WINDOW[res], shift,
                                              _l.darr(BOX), _l.iarr(N), r * x_n, x_n, _ptr(out), 8, 1, None))
            tol = 1e-12 * np.abs(want).max()
            np.testing.assert_allclose(_host(full), want, rtol=0, atol=tol, err_msg="%s shift %g full" % (res, shift))
            np.testing.assert_allclose(_host(out) - base, want, rtol=0, atol=tol, err_msg="%s shift %g P=%d" % (res, shift, P))


@pytest.mark.parametrize("N,P", [((45, 21, 35), 3), ((48, 36, 17), 4), ((30, 33, 16), 2)])
@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_ylm_mul_real_x_slabs(cuda, N, P, dtype):
    _l = _lib()
    rng = np.random.RandomState(71)
    field = rng.standard_normal(N).astype(dtype)
    C = np.array([10., -20., 5.])
    offset = C + 0.5 * np.asarray(BOX) / np.asarray(N)
    xg = [x.astype("f8") + offset[i] for i, x in enumerate(co.x_coords(N, BOX, "f8"))]
    xn = np.sqrt(sum(x ** 2 for x in xg))
    xhat = [x / xn for x in xg]
    x_n = N[0] // P
    tol = 1e-13 if dtype == "f8" else 2e-6
    for l, m in [(1, -1), (2, 1), (3, 0), (4, -3)]:
        want = field.astype("f8") * _ylm(l, m, xhat)
        outs = []
        for r, s in enumerate(ml.split_x(field, P)):
            a, b = _dev(s), _dev(np.zeros_like(s))
            _l.check(_l.lib().nbk_ylm_mul_real(_ptr(a), _ptr(b), _code(dtype), l, m, _l.iarr(N), _l.darr(BOX),
                                               _l.darr(offset), r * x_n, x_n, None))
            outs.append(_host(b))
        _close(np.concatenate(outs), want, tol)


# ---------------------------------------------------------------------------------------------
# E. tiled paint at cell boundaries
# ---------------------------------------------------------------------------------------------
PAINT_N = (48, 64, 80)
PAINT_BOXES = {"margin": (100., 3.3, 7000.), "pow2": (96., 64., 40.)}


def _pm(N, L, dtype="f8"):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.pmesh.pm import ParticleMesh
    return ParticleMesh(BoxSize=L, Nmesh=N, dtype=dtype, comm=SelfComm())


def _cell_order(pos, N, L, res):
    c = np.stack([ml.exact_cell(pos[:, d], N[d], L[d], res) % N[d] for d in range(3)], axis=1)
    return np.lexsort((c[:, 2], c[:, 1], c[:, 0]))


@pytest.mark.parametrize("box", sorted(PAINT_BOXES))
@pytest.mark.parametrize("pos_dtype", ["f4", "f8"])
@pytest.mark.parametrize("resampler", ["nnb", "cic", "tsc", "pcs"])
def test_tiled_paint_cell_boundaries(cuda, monkeypatch, box, pos_dtype, resampler):
    """NNB with unit mass is exact (every deposit 2^31 of M = 1): one particle in the wrong tile or cell fails;
    cell index bit-exact; both bucketing plans, cell-sorted and random order, shift 0 / 0.5, the interlaced pair"""
    from nbodykit_b200.pmesh.pm import RealField
    N, L = PAINT_N, PAINT_BOXES[box]
    pos, _ = ml.boundary_positions(N, L, pos_dtype, seed=5)
    pm = _pm(N, L)
    orders = {"cell-sorted": _cell_order(pos, N, L, resampler),
              "random": np.random.RandomState(6).permutation(len(pos))}
    want = {s: po.paint(pos, None, N, L, resampler, s) for s in (0.0, 0.5)}

    def check(got, w, what, direct=False):
        if resampler == "nnb":
            assert np.array_equal(got, w), what
        else:
            np.testing.assert_allclose(got, w, rtol=0, atol=(1e-12 if direct else 1e-7) * np.abs(w).max(), err_msg=what)
    for shift, w in want.items():
        assert np.array_equal(pm.cell_index(pos, resampler, shift).cpu().numpy(), po.cell_index(pos, N, L, resampler, shift))
        tr = pm.affine.shift(shift) if shift else None
        check(pm.paint(pos, resampler=resampler, transform=tr, method='direct').numpy(), w, "direct", direct=True)
        check(pm.paint(pos, resampler=resampler, transform=tr).numpy(), w, "default dispatch")
    for plan in ("coherent", "scattered"):
        monkeypatch.setenv("NBK_PAINT_BUCKET", plan)
        for oname, idx in orders.items():
            for shift, w in want.items():
                tr = pm.affine.shift(shift) if shift else None
                got = pm.paint(pos[idx], resampler=resampler, transform=tr, method='tiled').numpy()
                check(got, w, "%s %s shift %g" % (plan, oname, shift))
        r1, r2 = RealField(pm), RealField(pm)
        pm.paint_interlaced(pos, None, resampler, r1, r2, method='tiled', hold=False)
        check(r1.numpy(), want[0.0], "%s interlaced 1" % plan)
        check(r2.numpy(), want[0.5], "%s interlaced 2" % plan)


# ---------------------------------------------------------------------------------------------
# F. the fixed-point contract of the tiled paint
# ---------------------------------------------------------------------------------------------
def _masses(kind, n, seed=9):
    rng = np.random.RandomState(seed)
    if kind == "zero":
        return np.zeros(n)
    if kind == "negative":
        return -rng.uniform(0.1, 5.0, size=n)
    if kind == "span":
        return 10.0 ** rng.uniform(-6, 3, size=n) * rng.choice([-1.0, 1.0], size=n)
    # pow2-<where>-<dtype>: masses below 8, the largest at 8, just below or just above it in that dtype
    _, where, dt = kind.split("-")
    m = rng.uniform(0.0, 8.0, size=n).astype(dt)
    top = np.asarray(8.0, dtype=dt)
    if where != "at":
        top = np.nextafter(top, np.asarray(np.inf if where == "above" else 0.0, dtype=dt))
    m[rng.randint(0, n, size=50)] = top
    return m


MASS_SETS = ["pow2-at-f8", "pow2-below-f8", "pow2-above-f8", "pow2-at-f4", "pow2-below-f4", "pow2-above-f4", "negative",
             "zero", "span"]


@pytest.mark.parametrize("masses", MASS_SETS)
@pytest.mark.parametrize("resampler", ["nnb", "cic", "tsc", "pcs"])
def test_tiled_paint_fixed_point(cuda, masses, resampler):
    """NNB: bit-exact round-half-even(m 2^31 / M) sums (pins the scale M); other windows: per cell within the sum over
    its deposits of M 2^-32 + |m| 3 c 2^-28 -- an error relative to max |mass|, not to the cell"""
    N, L = PAINT_N, PAINT_BOXES["margin"]
    pos, _ = ml.boundary_positions(N, L, "f4", seed=10)
    mass = _masses(masses, len(pos))
    pm = _pm(N, L)
    got = pm.paint(pos, mass=mass, resampler=resampler, method='tiled').numpy()
    if resampler == "nnb":
        assert np.array_equal(got, ml.nnb_fixed_point(pos, mass, N, L))
    want = po.paint(pos, mass, N, L, resampler)
    bound, _ = ml.deposit_bound(pos, mass, N, L, resampler)
    err = np.abs(got - want)
    worst = np.argmax(err - bound)
    assert (err <= bound).all(), "worst cell: err %g > bound %g" % (err.flat[worst], bound.flat[worst])
