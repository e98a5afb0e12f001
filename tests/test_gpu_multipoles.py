"""
The multipole machinery of the Fourier-space path against float64 NumPy references (oracle/pmesh_oracle.py,
mesh_layouts.py, convpower_oracle.py):

A. every k_power_bin instance (2 dtypes x NELL = 1..8 x {LEAN, shared, global accumulators} x {SYM, oblique}: 96
   kernels), on every virtual-rank layout, at odd and Nyquist-carrying sides; one mesh with more rows than resident
   warps; multipoles up to the ABI limit l = 64 (Legendre weights from scipy.special.eval_legendre above l = 8, where
   the Horner form of the poly1d weights loses digits);
B. more than eight poles in FFTPower and FFTCorr (binned in groups of eight), on one rank and on two gloo ranks;
C. the real spherical harmonics kernels at every (l, m) of the l <= 8 table, on every layout, and ConvolvedFFTPower
   at l = 5 .. 8, on the global accumulators with the mirror field, and its refusal of l = 9.
"""
import numpy as np
import pytest
from gpu_helpers import code as _code, dev as _dev, host as _host, nbk as _lib, ptr as _p
from test_gpu_mesh_layouts import BOX, LAYOUT_FULLZ, LAYOUT_TRANSPOSED, SIDES, _bin, _layouts, _stat
from test_gpu_rank_statistics import _real_bin
from test_gpu_slab_route import _spawn

from oracle import convpower_oracle as co
from oracle import mesh_layouts as ml
from oracle import pmesh_oracle as po

pytestmark = pytest.mark.gpu

MAX_ELL, SMEM_LIMIT = 8, 200 * 1024


def _eval_legendre(ell, mu):
    from scipy.special import eval_legendre
    return eval_legendre(ell, mu)


# ---------------------------------------------------------------------------------------------
# A. every binning instance
# ---------------------------------------------------------------------------------------------
def _instance(dtype, kedges, muedges, ells, los, kind, coord):
    """the k_power_bin<T, NELL, SMEM_ACC, SYM, LEAN> instance launch_bin (csrc/binning.cu) picks, restated on the host:
    (dtype, NELL, 'lean' | 'shared' | 'global', sym).  The accumulators are shared when the edges and the per-bin
    sums fit in 200 KB; LEAN is the shared-accumulator auto power of a Hermitian complex field in float32
    coordinates; SYM is a line of sight along z."""
    Nx, Nmu, nell = len(kedges) - 1, len(muedges) - 1, len(ells)
    nb = (Nx + 2) * (Nmu + 2)
    edge_bytes = 8 * (Nx + 1 + Nmu + 1)
    acc_bytes = nb * (8 * (2 + 2 * nell) + 4)
    smem = edge_bytes + acc_bytes <= SMEM_LIMIT
    lean = smem and kind == "auto" and coord == 4           # (complex, hermitian = 1, no second or mirror field)
    sym = los[0] == 0.0 and los[1] == 0.0
    return (dtype, nell, "lean" if lean else ("shared" if smem else "global"), sym)


def _fourier_edges(N, Nmu, fine):
    Lv = np.asarray(BOX)
    dk = 2 * np.pi / Lv.min()
    kmax = np.pi * min(N) / Lv.max() + dk / 2
    step = dk / 8 if fine else dk
    return np.arange(0., kmax, step), np.linspace(-1, 1, Nmu + 1)


def _real_edges(N, Nmu, fine):
    dr = min(BOX) / max(N)
    step = dr / 8 if fine else dr
    return np.arange(0., 0.5 * min(BOX) + dr / 2, step), np.linspace(0, 1, Nmu + 1)


# the statistics of the shared / global slots, in turn: cross power with a compensation pair (f8 coordinates), the
# 3-D statistic itself (f4 coordinates, f8 mu), the anti-Hermitian fold, a cross power with the mirror field of
# nbk_power_bin2, the full-z layout with hermitian = 0, a real statistic on x slabs (FFTCorr), the auto power in f8
# coordinates (the general instance with an imaginary part known to vanish)
KINDS = ["cross", "p3d", "anti", "mirror", "fullz", "real", "auto8"]
OBLIQUE = [(0.6, 0., 0.8), (0., 1., 0.), (0.48, 0.6, 0.64)]
COMPS = [(None, None), ("CompensateTSCShotnoise",) * 2, ("CompensateCIC", "CompensatePCSShotnoise")]


def _ells(kind, nell, i):
    """l = 0 first; odd multipoles where the statistic has them, up to l = 24 in some of the slots"""
    if kind in ("auto", "auto8"):
        seq = list(range(0, 2 * nell, 2)) if i % 2 else [0, 2, 4, 8, 12, 16, 20, 24][:nell]
    elif kind == "p3d":
        seq = [0, 3, 6, 9, 12, 15, 18, 21][:nell]
    else:
        seq = list(range(nell))
    return seq


def _make_case(dtype, nell, acc, sym, i):
    kind = "auto" if acc == "lean" else KINDS[i % len(KINDS)]
    N = SIDES[i % len(SIDES)]
    los = (0., 0., 1.) if sym else OBLIQUE[i % len(OBLIQUE)]
    coord = {"cross": 8, "p3d": 48, "auto8": 8}.get(kind, 4)
    comp = COMPS[i % len(COMPS)] if kind in ("auto", "auto8", "cross") else (None, None)
    if kind == "auto":
        comp = (comp[0], comp[0])
    edges_fn = _real_edges if kind == "real" else _fourier_edges
    if acc == "global":
        for Nmu in (60, 100, 160, 240):          # fine k edges, many mu bins: the sums outgrow shared memory
            edges = edges_fn(N, Nmu, True)
            if _instance(dtype, edges[0], edges[1], [0] * nell, los, kind, coord)[2] == "global":
                break
    else:
        edges = edges_fn(N, 1 + i % 5, False)
    return dict(kind=kind, N=N, dtype=dtype, los=los, coord=coord, comp=comp, edges=edges, ells=_ells(kind, nell, i),
                clear=(i % 4 != 1))


def _case_table():
    cases, i = {}, 0
    for dtype in ("f8", "f4"):
        for nell in range(1, MAX_ELL + 1):
            for sym in (True, False):
                for acc in ("lean", "shared", "global"):
                    c = _make_case(dtype, nell, acc, sym, i)
                    cases["%s-n%d-%s-%s-%s" % (dtype, nell, acc, "sym" if sym else "obl", c["kind"])] = c
                    i += 1
    return cases


CASES = _case_table()
# more rows than an H100 holds resident warps (132 SMs x 64): the persistent row loop of every warp runs more than once
CASES["wave-oblique-lean"] = dict(kind="auto", N=(160, 144, 30), dtype="f8", los=(0.6, 0., 0.8), coord=4,
                                  comp=("CompensateCICShotnoise",) * 2, edges=_fourier_edges((160, 144, 30), 3, False),
                                  ells=[0, 2, 4], clear=True)
CASES["wave-oblique-global-mirror"] = dict(kind="mirror", N=(160, 144, 30), dtype="f8", los=(0., 1., 0.), coord=4,
                                           comp=(None, None), edges=_fourier_edges((160, 144, 30), 60, True),
                                           ells=[0, 1, 2, 3], clear=True)
# the largest multipole the C ABI takes
CASES["ell64-z"] = dict(kind="cross", N=(44, 52, 37), dtype="f8", los=(0., 0., 1.), coord=8, comp=(None, None),
                        edges=_fourier_edges((44, 52, 37), 4, False), ells=[0, 31, 64], clear=True)
CASES["ell64-oblique-anti"] = dict(kind="anti", N=(45, 21, 35), dtype="f8", los=(0.48, 0.6, 0.64), coord=4,
                                   comp=(None, None), edges=_fourier_edges((45, 21, 35), 3, False), ells=[0, 63, 64],
                                   clear=True)


def _case_instance(c):
    return _instance(c["dtype"], c["edges"][0], c["edges"][1], c["ells"], c["los"], c["kind"], c["coord"])


def test_case_table_covers_every_instance():
    """the table reaches each of the 96 instances launch_bin can pick (the check runs without a GPU, but the module
    is GPU-marked: it is asserted again by every case below)"""
    want = {(d, n, a, s) for d in ("f8", "f4") for n in range(1, MAX_ELL + 1) for a in ("lean", "shared", "global")
            for s in (True, False)}
    got = {_case_instance(c) for c in CASES.values()}
    assert len(want) == 96
    assert want <= got, "instances no case reaches: %s" % sorted(want - got)
    kinds = {c["kind"] for c in CASES.values()}
    assert kinds == {"auto"} | set(KINDS)
    assert {c["coord"] for c in CASES.values()} == {4, 8, 48}


def _fields(c):
    """device inputs (host arrays, per layout split) and the float64 statistics the reference bins:
    (arrays, [(y3d, x3d, hermitian_symmetric, sign(ell))], los for the oracle)"""
    N, dtype, kind, comp = c["N"], c["dtype"], c["kind"], c["comp"]
    rng = np.random.RandomState(sum(N) + len(c["ells"]))
    V = float(np.prod(BOX))
    los = c["los"]
    if kind == "real":
        y = rng.standard_normal(N).astype(dtype)
        return [y], [(y.astype("f8"), co.x_coords(N, BOX, "f4"), False, None)], list(los)
    if kind == "fullz":
        _, f1 = ml.spectra(N, rng, dtype)
        _, f2 = ml.spectra(N, rng, dtype)
        y = f1.astype("c16") * np.conj(f2.astype("c16")) * V
        if c["clear"]:
            y[0, 0, 0] = 0
        return [f1, f2], [(y, ml.k_coords(N, BOX, "f4", fullz=True), False, None)], list(los)
    c1, _ = ml.spectra(N, rng, dtype)
    c2 = ml.spectra(N, rng, dtype)[0] if kind in ("cross", "anti", "mirror") else None
    if c["coord"] == 8:
        x3d, los_o = po.k_coords(N, BOX, "f8"), list(los)
    elif c["coord"] == 48:
        x3d, los_o = po.k_coords(N, BOX, "f4"), np.asarray(los, dtype="f8")     # numpy-scalar los: f8 mu
    else:
        x3d, los_o = po.k_coords(N, BOX, "f4"), list(los)
    if kind == "p3d":
        return [c1], [(c1.astype("c16"), x3d, True, None)], los_o
    if kind == "mirror":
        # the stored mode k: c1 conj(c2) V; its unstored mirror -k (for 0 < jz): conj(c1 conj(c3)) V, binned at the
        # k and mu of k with Leg_l(-mu) = (-1)^l Leg_l(mu)
        c3 = ml.spectra(N, rng, dtype)[0]
        a, b, m = c1.astype("c16"), c2.astype("c16"), c3.astype("c16")
        y1 = a * np.conj(b) * V
        if c["clear"]:
            y1[0, 0, 0] = 0
        jz = po.freq_index(int(N[2]), compressed=True)
        y2 = np.conj(a * np.conj(m)) * V * (jz > 0)
        return [c1, c2, c3], [(y1, x3d, False, None), (y2, x3d, False, "odd")], los_o
    y = _stat(c1, c2, N, "cross" if c2 is not None else "auto", V, c["clear"], comp)
    return [c1] + ([c2] if c2 is not None else []), [(y, x3d, True, None)], los_o


def _reference(c, parts, los_o):
    """raw sums (nsum, xsum, musum, ysum[Nell]) and S_bin = sum over the bin of |statistic| x Hermitian weight"""
    ells, edges, kind = c["ells"], c["edges"], c["kind"]
    poles = ells[1:] if len(ells) > 1 else []
    leg = _eval_legendre if max(ells) > MAX_ELL else None
    n = x = mu = None
    ysum, S = 0, 0
    for y, x3d, herm, odd in parts:
        yy = 1j * y if kind == "anti" else y
        xs, ms, ys, ns = po.project_sums(yy, x3d, edges, los_o, poles, hermitian_symmetric=herm, legendre=leg)
        if kind == "anti":
            ys = -1j * ys
        if odd:
            ys = ys * np.array([(-1.0) ** l for l in ells]).reshape(-1, 1, 1)
        ysum = ysum + ys
        S = S + po.project_sums(np.abs(y), x3d, edges, los_o, [], hermitian_symmetric=herm)[2][0].real
        if n is None:
            n, x, mu = ns, xs, ms
    if kind == "mirror":      # counts, k and mu sums with the Hermitian weights of the compressed layout
        x, mu, _, n = po.project_sums(np.zeros_like(parts[0][0]), parts[0][1], edges, los_o, [])
    return (n, x, mu, ysum), S


def _layout_sums(c, arrays):
    """(layout label, raw sums summed over the virtual ranks) for every layout of the case"""
    N, dtype, kind = c["N"], c["dtype"], c["kind"]
    ells, edges, los = c["ells"], c["edges"], c["los"]
    if kind == "real":
        for P in [1] + ml.rank_counts(N[0]):
            x_n, tot = N[0] // P, None
            for r, s in enumerate(ml.split_x(arrays[0], P)):
                got = _real_bin(_dev(s), N, dtype, r * x_n, x_n, edges, los, ells)
                tot = got if tot is None else tuple(a + b for a, b in zip(tot, got))
            yield "x slabs P=%d" % P, tot
        return
    herm = 0 if kind == "fullz" else (2 if kind == "anti" else 1)
    bits = LAYOUT_FULLZ if kind == "fullz" else 0
    kw = dict(edges=edges, los=los, ells=ells, herm=herm, coord=c["coord"], is_p3d=(kind == "p3d"),
              V=float(np.prod(BOX)), clear=c["clear"], comp=c["comp"])
    for P in _layouts(N):
        if P == 0:
            yield "P=0", _bin([_dev(a) for a in arrays], N, dtype, bits, 0, N[0], **kw)
            continue
        y_n, tot = N[1] // P, None
        for r, parts in enumerate(zip(*[ml.split_transposed(a, P) for a in arrays])):
            s = _bin([_dev(a) for a in parts], N, dtype, bits | LAYOUT_TRANSPOSED, r * y_n, y_n, **kw)
            tot = s if tot is None else tuple(a + b for a, b in zip(tot, s))
        yield "P=%d" % P, tot


def _check_case(cid, c):
    arrays, parts, los_o = _fields(c)
    (nw, xw, mw, yw), S = _reference(c, parts, los_o)
    tol = 1e-12 if c["dtype"] == "f8" else 2e-6
    ells = c["ells"]
    nb = nw.size
    yw = yw.reshape(len(ells), nb)
    # |sum_bin (2l+1) Leg_l(mu) y w_H| <= (2l+1) S_bin: the error of a sum that cancels is bounded by that, not by the
    # sum itself
    bound = tol * np.array([2 * l + 1 for l in ells]).reshape(-1, 1) * S.reshape(1, nb)
    for what, (ng, xg, mg, yg) in _layout_sums(c, arrays):
        tag = "%s %s" % (cid, what)
        assert np.array_equal(ng, nw.reshape(-1)), "%s: mode counts differ" % tag
        for g, w, name in ((xg, xw, "k sums"), (mg, mw, "mu sums")):
            w = w.reshape(-1)
            np.testing.assert_allclose(g, w, rtol=tol, atol=tol * max(np.abs(w).max(), 1e-300), err_msg="%s %s" % (tag, name))
        err = np.abs(yg - yw)
        lim = tol * np.abs(yw) + bound
        if not (err <= lim).all():
            il, ib = np.unravel_index(np.argmax(err - lim), err.shape)
            raise AssertionError("%s: l=%d bin %d: got %r, want %r (S_bin %g)" % (tag, ells[il], ib, yg[il, ib],
                                                                                   yw[il, ib], S.reshape(-1)[ib]))


@pytest.mark.parametrize("cid", sorted(CASES))
def test_power_bin_instance(cuda, cid):
    """counts bit for bit, k / mu sums to tol, every multipole sum within tol (2l+1) S_bin of the float64 reference
    (tol 1e-12 for f8 fields, 2e-6 for f4), on every layout"""
    _check_case(cid, CASES[cid])


def test_power_bin_rejects_ell_65(cuda):
    c = dict(CASES["ell64-z"], ells=[0, 65])
    arrays, _, _ = _fields(c)
    with pytest.raises(_lib().NbkError, match="bad multipole 65"):
        next(_layout_sums(c, arrays))


# ---------------------------------------------------------------------------------------------
# B. more than eight poles
# ---------------------------------------------------------------------------------------------
MANY_N, MANY_L = (32, 36, 30), (100., 130., 70.)
MANY_POLES = {"even16": list(range(0, 17, 2)), "all12": list(range(13))}
MANY_LOS = {"z": [0, 0, 1], "oblique": [0.6, 0, 0.8]}


def _many_field():
    return np.random.RandomState(17).standard_normal(MANY_N)


def _fftpower(comm, field, poles, los):
    from nbodykit_b200.lab import ArrayMesh, FFTPower
    r = FFTPower(ArrayMesh(field, BoxSize=MANY_L, comm=comm), mode="2d", Nmu=4, poles=poles, los=los)
    out = {"power." + v: np.array(r.power[v]) for v in r.power.variables}
    out.update({"poles." + v: np.array(r.poles[v]) for v in r.poles.variables})
    return out


@pytest.mark.parametrize("los", sorted(MANY_LOS))
@pytest.mark.parametrize("pid", sorted(MANY_POLES))
def test_fftpower_more_than_eight_poles(cuda, pid, los):
    """FFTPower mode='2d' on an ArrayMesh with 9 or 13 poles, against r2c + project_to_basis with exact Legendre
    weights"""
    from nbodykit_b200.comm import SelfComm
    poles, lv = MANY_POLES[pid], MANY_LOS[los]
    field = _many_field()
    got = _fftpower(SelfComm(), field, poles, lv)
    N, L = np.asarray(MANY_N), np.asarray(MANY_L)
    c = po.r2c(field)
    y = c * np.conj(c) * L.prod()
    y[0, 0, 0] = 0
    dk = 2 * np.pi / L.min()
    edges = [np.arange(0., np.pi * N.min() / L.max() + dk / 2, dk), np.linspace(-1, 1, 5)]
    (xm, mm, y2d, n2d), (k1, pw, n1) = po.project_to_basis(y, po.k_coords(N, L, "f4"), edges, lv, poles,
                                                           legendre=_eval_legendre)
    assert np.array_equal(got["power.modes"], n2d) and np.array_equal(got["poles.modes"], n1)
    np.testing.assert_allclose(got["poles.k"], k1, rtol=1e-12)
    scale = np.nanmax(np.abs(pw[0]))
    np.testing.assert_allclose(got["power.power"], y2d, rtol=1e-9, atol=1e-9 * scale)
    for i, ell in enumerate(poles):
        np.testing.assert_allclose(got["poles.power_%d" % ell], pw[i], rtol=1e-9, atol=1e-9 * scale,
                                   err_msg="l=%d" % ell)
    # every even multipole carries signal, so a pole binned into the wrong row would show
    assert all(np.nanmax(np.abs(pw[i])) > 1e-6 * scale for i, ell in enumerate(poles) if not ell % 2)


@pytest.mark.parametrize("los", sorted(MANY_LOS))
def test_fftpower_more_than_eight_poles_two_ranks(cuda, los):
    """the grouped binning all-reduces once: two gloo ranks equal one"""
    from nbodykit_b200.comm import SelfComm
    poles, lv = MANY_POLES["all12"], MANY_LOS[los]
    field = _many_field()
    one = _fftpower(SelfComm(), field, poles, lv)
    for r, part in enumerate(_spawn(_fftpower, 2, field, poles, lv)):
        assert sorted(part) == sorted(one)
        scale = np.nanmax(np.abs(one["poles.power_0"]))
        for key in sorted(one):
            if key.endswith("modes"):
                assert np.array_equal(part[key], one[key]), "rank %d %s" % (r, key)
            else:
                np.testing.assert_allclose(part[key], one[key], rtol=1e-12, atol=1e-12 * scale,
                                           err_msg="rank %d %s" % (r, key))


def test_fftcorr_nine_poles(cuda):
    """FFTCorr with 9 poles: the real-input binning in groups, against c2r + project_to_basis"""
    from nbodykit_b200.lab import ArrayMesh, FFTCorr
    poles = list(range(0, 17, 2))
    field = _many_field()
    N, L = np.asarray(MANY_N), np.asarray(MANY_L)
    r = FFTCorr(ArrayMesh(field, BoxSize=MANY_L), mode="2d", Nmu=4, poles=poles, los=[0.6, 0, 0.8])
    c = po.r2c(field)
    p3d = c * np.conj(c) * L.prod()
    p3d[0, 0, 0] = 0
    xi = po.c2r(p3d, N) / L.prod()
    dr = L.min() / N.max()
    edges = [np.arange(0., 0.5 * L.min() + dr / 2, dr), np.linspace(0, 1, 5)]
    (xm, mm, y2d, n2d), (r1, pw, n1) = po.project_to_basis(xi, co.x_coords(N, L, "f4"), edges, [0.6, 0, 0.8], poles,
                                                           hermitian_symmetric=False, legendre=_eval_legendre)
    assert np.array_equal(r.corr["modes"], n2d) and np.array_equal(r.poles["modes"], n1)
    scale = np.nanmax(np.abs(pw[0]))
    np.testing.assert_allclose(r.corr["corr"], y2d.real, rtol=1e-9, atol=1e-9 * scale)
    for i, ell in enumerate(poles):
        np.testing.assert_allclose(r.poles["corr_%d" % ell], pw[i].real, rtol=1e-9, atol=1e-9 * scale,
                                   err_msg="l=%d" % ell)


# ---------------------------------------------------------------------------------------------
# C. Y_lm up to the table's limit
# ---------------------------------------------------------------------------------------------
YLM_LM = [(l, m) for l in range(MAX_ELL + 1) for m in range(-l, l + 1)]


def _ylm(l, m, d):
    return co.real_ylm(l, m, d[0], d[1], d[2])


def _close(got, want, tol, what):
    err = np.abs(got - want).max()
    assert err <= tol * np.abs(want).max(), "%s: max error %g > %g x max |want| %g" % (what, err, tol, np.abs(want).max())


@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_ylm_mul_real_every_lm(cuda, dtype):
    """nbk_ylm_mul_real on x slabs (P = 1, 3) for every (l, m) with l <= 8"""
    _l = _lib()
    N, P = (45, 21, 35), 3
    field = np.random.RandomState(71).standard_normal(N).astype(dtype)
    offset = np.array([10., -20., 5.]) + 0.5 * np.asarray(BOX) / np.asarray(N)
    xg = [x.astype("f8") + offset[i] for i, x in enumerate(co.x_coords(N, BOX, "f8"))]
    xn = np.sqrt(sum(x ** 2 for x in xg))
    xhat = [x / xn for x in xg]
    tol = 1e-13 if dtype == "f8" else 2e-6
    for l, m in YLM_LM:
        want = field.astype("f8") * _ylm(l, m, xhat)
        for p in (1, P):
            x_n, outs = N[0] // p, []
            for r, s in enumerate(ml.split_x(field, p)):
                a, b = _dev(s), _dev(np.zeros_like(s))
                _l.check(_l.lib().nbk_ylm_mul_real(_p(a), _p(b), _code(dtype), l, m, _l.iarr(N), _l.darr(BOX),
                                                   _l.darr(offset), r * x_n, x_n, None), "nbk_ylm_mul_real")
                outs.append(_host(b))
            _close(np.concatenate(outs), want, tol, "l=%d m=%d P=%d" % (l, m, p))


def _dirs(N, fullz):
    """(khat, the direction of the unstored mirror mode) on the compressed or full-z layout, f8, khat := 0 at k = 0:
    every component flips sign except at a Nyquist index, whose label stays -N/2"""
    if not fullz:
        return ml.mirror_dirs(N, BOX)
    k = ml.k_coords(N, BOX, "f8", fullz=True)
    m = []
    for d in range(3):
        j = po.freq_index(int(N[d]))
        keep = (2 * j == -int(N[d])).reshape(k[d].shape)
        m.append(np.where(keep, k[d], -k[d]))
    kn = np.sqrt(sum(x ** 2 for x in k))
    inv = np.where(kn == 0, 0.0, 1.0 / np.where(kn == 0, 1.0, kn))
    return [x * inv for x in k], [x * inv for x in m]


@pytest.mark.parametrize("N", [(44, 52, 37), (48, 36, 16)])
@pytest.mark.parametrize("dtype", ["f8", "f4"])
def test_ylm_mul_complex_acc_every_lm(cuda, N, dtype):
    """nbk_ylm_mul_complex_acc and _acc2 (with the mirror direction, Nyquist labels kept) for every (l, m) with
    l <= 8, on every transposed y-slab split and on the full-z layout; accumulating onto a non-zero field"""
    _l = _lib()
    rng = np.random.RandomState(72)
    c, full = ml.spectra(N, rng, dtype)
    base, base_f = ml.spectra(N, rng, dtype)
    tol = 1e-13 if dtype == "f8" else 2e-6
    cd = "c16"
    for fullz in (False, True):
        khat, mhat = _dirs(N, fullz)
        src, acc0 = (full, base_f) if fullz else (c, base)
        layouts = [0] if fullz else _layouts(N)
        bits = LAYOUT_FULLZ if fullz else 0
        for l, m in YLM_LM:
            want_a = acc0.astype(cd) + src.astype(cd) * _ylm(l, m, khat)
            want_b = acc0.astype(cd) + src.astype(cd) * _ylm(l, m, mhat)
            for P in layouts:
                pieces = [(acc0, acc0, acc0, src)] if P == 0 else \
                    list(zip(*[ml.split_transposed(a, P) for a in (acc0, acc0, acc0, src)]))
                outs = []
                for r, (a1, a2, b2, s) in enumerate(pieces):
                    ts = [_dev(a) for a in (a1, a2, b2, s)]
                    lay, start, count = (bits, 0, N[0]) if P == 0 else (bits | LAYOUT_TRANSPOSED, r * (N[1] // P),
                                                                       N[1] // P)
                    _l.check(_l.lib().nbk_ylm_mul_complex_acc(_p(ts[0]), _p(ts[3]), _code(dtype), l, m, _l.iarr(N),
                                                              _l.darr(BOX), lay, start, count, None))
                    _l.check(_l.lib().nbk_ylm_mul_complex_acc2(_p(ts[1]), _p(ts[2]), _p(ts[3]), _code(dtype), l, m,
                                                               _l.iarr(N), _l.darr(BOX), lay, start, count, None))
                    outs.append([_host(t) for t in ts[:3]])
                if P == 0:
                    a1, a2, b2 = outs[0]
                else:
                    a1, a2, b2 = [ml.join_transposed([o[i] for o in outs]) for i in range(3)]
                what = "l=%d m=%d P=%d fullz=%s" % (l, m, P, fullz)
                _close(a1, want_a, tol, what + " acc")
                _close(a2, want_a, tol, what + " acc2")
                _close(b2, want_b, tol, what + " acc2 mirror")
                # k = 0: khat := 0, only the constant term of the polynomial is left
                want0 = acc0.flat[0].astype(cd) + src.flat[0].astype(cd) * float(co.real_ylm(l, m, 0., 0., 0.))
                assert abs(a1.flat[0] - want0) <= tol * max(abs(want0), 1e-300) + 1e-300, what + " k = 0"


def _fkp(box=512.):
    from test_gpu_convpower import _fkp as fkp
    return fkp(box=box)


def _conv_args(d, r, mesh, poles):
    from test_gpu_convpower import NBAR
    wfd = 1. / (1 + 1e4 * NBAR)
    return (np.asarray(d['Position']), np.asarray(r['Position']), (np.asarray(d['Weight']), wfd * np.ones(d.size)),
            (np.ones(r.size), wfd * np.ones(r.size)), NBAR * np.ones(d.size), NBAR * np.ones(r.size), 32,
            mesh.attrs['BoxSize'], mesh.attrs['BoxCenter'], poles)


def _conv_check(res, o, poles, imag=True):
    assert np.array_equal(res.poles['modes'], o['modes'])
    np.testing.assert_allclose(res.poles['k'], o['k'], rtol=1e-6, equal_nan=True)
    scale = np.nanmax(np.abs(o['power_0']))
    for ell in poles:
        got, want = res.poles['power_%d' % ell], o['power_%d' % ell]
        for part in ("real", "imag") if imag else ("real",):
            np.testing.assert_allclose(np.nan_to_num(getattr(got, part)), np.nan_to_num(getattr(want, part)), rtol=1e-5,
                                       atol=2e-6 * scale, err_msg="l=%d %s" % (ell, part))


CONV_POLES = [0, 5, 6, 7, 8]


def test_convolved_power_high_ells_complex_mesh(cuda):
    """'c16' mesh (mirror accumulator, anti-Hermitian fold of l = 5, 7) against the full complex-mesh restatement"""
    from nbodykit_b200.lab import ConvolvedFFTPower
    fkp, d, r = _fkp()
    mesh = fkp.to_mesh(Nmesh=32)
    assert mesh.complex_mesh
    res = ConvolvedFFTPower(mesh, poles=CONV_POLES, dk=0.02)
    o = co.convpower_full(*_conv_args(d, r, mesh, CONV_POLES), dk=0.02)
    _conv_check(res, o, CONV_POLES)


def test_convolved_power_high_ells_f8_mesh(cuda):
    from nbodykit_b200.lab import ConvolvedFFTPower
    fkp, d, r = _fkp()
    mesh = fkp.to_mesh(Nmesh=32, dtype='f8', resampler='tsc')
    res = ConvolvedFFTPower(mesh, poles=CONV_POLES, dk=0.02)
    o = co.convpower(*_conv_args(d, r, mesh, CONV_POLES), resampler='tsc', dk=0.02)
    _conv_check(res, o, CONV_POLES, imag=False)


def test_convolved_power_global_accumulators_mirror(cuda):
    """'c16' mesh with dk fine enough that the per-bin sums leave shared memory: the global-accumulator instance with
    the mirror field of nbk_power_bin2"""
    from nbodykit_b200.lab import ConvolvedFFTPower
    poles, dk = [0, 3, 8], 1e-4
    fkp, d, r = _fkp()
    mesh = fkp.to_mesh(Nmesh=32)
    L = mesh.attrs['BoxSize']
    kedges = np.arange(0., np.pi * 32 / L.max() + dk / 2, dk)
    assert _instance("f8", kedges, [-1, 1], [0, 8], (0., 0., 1.), "mirror", 4)[2] == "global"
    res = ConvolvedFFTPower(mesh, poles=poles, dk=dk)
    o = co.convpower_full(*_conv_args(d, r, mesh, poles), dk=dk)
    _conv_check(res, o, poles)


def test_convolved_power_refuses_ell_9_before_painting(cuda):
    from nbodykit_b200.lab import ConvolvedFFTPower
    fkp, _, _ = _fkp()
    mesh = fkp.to_mesh(Nmesh=32)
    n0 = _lib().launch_count()
    with pytest.raises(ValueError, match="l <= 8"):
        ConvolvedFFTPower(mesh, poles=[0, 2, 9])
    assert _lib().launch_count() == n0, "kernels ran before the multipole was refused"
