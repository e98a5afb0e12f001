"""
FFTPower, ConvolvedFFTPower, FFTCorr, ProjectedFFTPower, RealField.preview and MultipleSpeciesCatalog meshes on P ranks
of one GPU, against one rank and against float64 NumPy references (oracle/pmesh_oracle.py, convpower_oracle.py,
mesh_layouts.py).

A. P processes over gloo (127.0.0.1) share device 0 with the all-to-all transpose (NBK_FFT_TRANSPOSE=nccl).  Every rank
holds a share of every catalogue -- one split leaves a rank without rows, another hands every rank the rows of another
rank's slab, so that everything is routed -- and one spawn per mesh geometry computes every statistic.  The parent
computes the same statistics on one rank (SelfComm) from the whole catalogues and the float64 restatements of the
one-GPU tests (test_gpu_fftpower.py, test_gpu_convpower.py, test_gpu_meshapi.py).

B. The two layouts A reaches only through the whole pipeline, on P virtual ranks of one process: nbk_power_bin of a real
statistic on x slabs (FFTCorr's binning) and nbk_cross_power on transposed y slabs (FFTCorr's 3-D power, zero mode
cleared on the rank that owns it).
"""
import numpy as np
import pytest
from gpu_helpers import code as _code, dev as _dev, host as _host, nbk as _lib, ptr as _p
from test_gpu_mesh_layouts import BOX, SIDES, _check_sums
from test_gpu_slab_route import _spawn

from oracle import convpower_oracle as co
from oracle import mesh_layouts as ml
from oracle import pmesh_oracle as po

pytestmark = pytest.mark.gpu

# id: (Nmesh, BoxSize, P, catalogue split)
# 32^3: power-of-two FFT, x_n = 8 at P = 4 (interlaced TSC reaches past a slab); (48, 36, 30): mixed-radix sides, a
# non-cubic box and an odd Nzc = 16; (44, 22, 26): Bluestein sides (11, 13) on ranks
GEOMS = {"32-P2": ((32, 32, 32), (200., 200., 200.), 2, "empty"),
         "32-P4": ((32, 32, 32), (200., 200., 200.), 4, "remote"),
         "48x36x30-P3": ((48, 36, 30), (100., 130., 70.), 3, "empty"),
         "44x22x26-P2": ((44, 22, 26), (120., 70., 90.), 2, "remote")}
NMU, POLES, CONV_POLES = 4, [0, 2, 4], [0, 1, 2, 3, 4]
# the FKP survey volume: 0.8 of the box, off the origin (BoxCenter and the x-slab offset of Y_lm(xhat) both matter)
SHIFT = np.array([1000., -300., 700.])
# statistics formed from an f4 mesh
F4_STATS = ("cross-x", "cross-y")
# the fields are painted with the tiled fixed-point paint on one side and partly through the REDG ghost batches on the
# other: the statistics agree to a few quanta (2^-31 max|w| per deposit) x sqrt(deposits per cell), bounded by 2e-8 of
# max |stat| in f8 and 2e-5 in f4 (tests/mgpu_check.py)
TOL_F8, TOL_F4 = 2e-8, 2e-5


def _dk(L):
    return 2 * np.pi / max(L)


def _catalogues(N, L):
    """d1: f4 positions with weights; d2: f8 positions; fd / fr: FKP data and randoms in an off-origin survey volume,
    with a second, per-object FKP weight for the cross multipoles"""
    rng = np.random.RandomState(sum(N))
    L = np.asarray(L, dtype="f8")
    n1, n2, nd, nr = 20000, 12000, 6000, 30000
    vol = 0.8 ** 3 * L.prod()
    nbar = nd / vol
    cats = {"d1": {"Position": (rng.uniform(size=(n1, 3)) * L).astype("f4"), "Weight": rng.uniform(0.5, 1.5, size=n1)},
            "d2": {"Position": rng.uniform(size=(n2, 3)) * L}}
    for name, n in (("fd", nd), ("fr", nr)):
        cats[name] = {"Position": rng.uniform(size=(n, 3)) * 0.8 * L + 0.1 * L + SHIFT, "NZ": np.full(n, nbar),
                      "FKPWeight2": rng.uniform(0.3, 0.7, size=n)}
    cats["fd"]["Weight"] = rng.uniform(0.8, 1.2, size=nd)
    return cats, nbar


def _owners(cats, N, L, P, split):
    """the rank holding each row: 'empty' -- ranks 1 .. P-1 at random, rank 0 holds nothing; 'remote' -- rank r holds
    the rows of slab r + 1 (in the frame the rows are painted in: the FKP rows relative to the randoms' box centre)"""
    rng = np.random.RandomState(7)
    pr = cats["fr"]["Position"]
    centre = 0.5 * (pr.min(axis=0) + pr.max(axis=0))
    out = {}
    for name, cols in cats.items():
        x = cols["Position"][:, 0].astype("f8") - (centre[0] if name in ("fd", "fr") else 0.0)
        slab = (np.floor(x * (N[0] / L[0])).astype("i8") % N[0]) // (N[0] // P)
        out[name] = rng.randint(1, P, size=len(x)) if split == "empty" else (slab + 1) % P
    return out


def _put(out, name, stat):
    for var in stat.variables:
        out["%s.%s" % (name, var)] = np.array(stat[var])
    for dim in stat.dims:
        out["%s.edges_%s" % (name, dim)] = np.array(stat.edges[dim])


def _statistics(comm, gid, cats, owner, P0):
    """every statistic of geometry `gid` on this rank's rows, as numpy (real fields: this rank's x slab)"""
    import torch
    from nbodykit_b200.lab import (ArrayCatalog, ConvolvedFFTPower, FFTCorr, FFTPower, FKPCatalog, MultipleSpeciesCatalog,
                                   ProjectedFFTPower)
    N, L, _, _ = GEOMS[gid]
    dk = _dk(L)

    def cat(name):
        mine = slice(None) if comm.size == 1 else owner[name] == comm.rank
        cols = {k: torch.from_numpy(np.ascontiguousarray(v[mine])).cuda() for k, v in cats[name].items()}
        return ArrayCatalog(cols, comm=comm, BoxSize=L)
    out = {}
    d1, d2 = cat("d1"), cat("d2")

    # FFTPower: auto (TSC interlaced, compensated, f8), cross with one f4 and one f8 mesh along x and y, dk = 0
    mesh = d1.to_mesh(Nmesh=N, BoxSize=L, resampler="tsc", interlaced=True, compensated=True, dtype="f8")
    r = FFTPower(mesh, mode="2d", Nmu=NMU, poles=POLES, dk=dk)
    _put(out, "auto", r.power)
    _put(out, "auto-poles", r.poles)
    for key in ("N1", "N2", "shotnoise"):
        out["attr.auto." + key] = r.attrs[key]
    real = mesh.compute(mode="real")
    out["field.tsc"] = real.numpy()
    for tag, axes in (("0", [0]), ("2", [2]), ("20", [2, 0]), ("all", None)):
        out["preview%s.value" % tag] = np.asarray(real.preview(axes=axes))

    def cic(c, dtype):
        return c.to_mesh(Nmesh=N, BoxSize=L, resampler="cic", compensated=True, dtype=dtype)
    for name, los, (t1, t2) in (("cross-x", [1, 0, 0], ("f4", "f8")), ("cross-y", [0, 1, 0], ("f8", "f4"))):
        r = FFTPower(cic(d1, t1), second=cic(d2, t2), mode="2d", Nmu=NMU, poles=[0, 2], los=los, dk=dk)
        _put(out, name, r.power)
        _put(out, name + "-poles", r.poles)
        for key in ("N1", "N2", "shotnoise"):
            out["attr.%s.%s" % (name, key)] = r.attrs[key]
    r = FFTPower(cic(d1, "f8"), mode="1d", dk=0)
    _put(out, "dk0", r.power)

    # FFTCorr on the compensated CIC mesh: (r, mu) with poles, and one bin per distinct separation
    r = FFTCorr(cic(d1, "f8"), mode="2d", Nmu=NMU, poles=[0, 2])
    _put(out, "corr2d", r.corr)
    _put(out, "corr2d-poles", r.poles)
    out["attr.corr2d.N1"] = r.attrs["N1"]
    r = FFTCorr(cic(d1, "f8"), mode="1d", dr=0)
    _put(out, "corr-dr0", r.corr)

    # ProjectedFFTPower: x summed over (preview all-reduces the slabs) and x kept (preview gathers them)
    for tag, axes in (("1", [1]), ("01", [0, 1])):
        r = ProjectedFFTPower(d1, Nmesh=N, axes=axes)
        _put(out, "proj" + tag, r.power)

    # MultipleSpeciesCatalog mesh
    sp = MultipleSpeciesCatalog(["a", "b"], d1, d2).to_mesh(Nmesh=N, BoxSize=L, dtype="f8").compute(mode="real")
    out["field.species"] = sp.numpy()
    for key in ("N", "num_per_cell", "a.W", "b.W", "a.N", "b.N", "shotnoise"):
        out["attr.species." + key] = sp.attrs[key]

    # ConvolvedFFTPower: default 'c16' mesh (mirror accumulator), 'f8' mesh, and a cross with another FKP weight
    fkp = FKPCatalog(cat("fd"), cat("fr"), P0=P0)
    runs = (("conv-c16", dict(resampler="cic"), CONV_POLES, None),
            ("conv-f8", dict(resampler="tsc", dtype="f8"), CONV_POLES, None),
            ("conv-cross", dict(resampler="tsc", dtype="f8"), [0, 2], dict(resampler="tsc", dtype="f8",
                                                                           fkp_weight="FKPWeight2")))
    for name, kw, poles, kw2 in runs:
        second = None if kw2 is None else fkp.to_mesh(Nmesh=N, BoxSize=L, **kw2)
        r = ConvolvedFFTPower(fkp.to_mesh(Nmesh=N, BoxSize=L, **kw), poles=poles, second=second, dk=dk)
        _put(out, name, r.poles)
        for key in ("alpha", "data.norm", "randoms.norm", "shotnoise", "BoxCenter"):
            out["attr.%s.%s" % (name, key)] = np.asarray(r.attrs[key])

    # complex-dtype ParticleMesh is one-rank only
    if comm.size > 1:
        try:
            FFTPower(d1.to_mesh(Nmesh=N, BoxSize=L, dtype="c16"), mode="1d")
            out["c16-raises"] = False
        except NotImplementedError:
            out["c16-raises"] = True
    return out


# ---------------------------------------------------------------------------------------------
# comparisons
# ---------------------------------------------------------------------------------------------
def _var(key):
    return key.rsplit(".", 1)[1]


def _is_stat(key):
    return not key.startswith(("attr.", "field.")) and _var(key) not in ("modes", "k", "r", "mu") and \
        not _var(key).startswith("edges_")


def _stat_scale(one, key):
    """max |stat| over the whole statistic (its wedges and multipoles): the l > 0 multipoles and the wedges are sums
    with cancellations, their errors follow the amplitude of the monopole"""
    group = key.split(".")[0].replace("-poles", "")
    vals = [np.nanmax(np.abs(v)) for k, v in one.items() if _is_stat(k) and k.split(".")[0].replace("-poles", "") == group]
    return max(vals)


def _vs_one(got, want, key, what, scale=None):
    """one entry of a P-rank result against one rank; `scale` bounds the error of a statistic (default max |want|)"""
    g, w = np.asarray(got), np.asarray(want)
    tag = "%s %s" % (what, key)
    assert g.shape == w.shape, tag
    v = _var(key)
    if v == "modes" or v.startswith("edges_") or g.dtype.kind in "iub":
        np.testing.assert_array_equal(g, w, err_msg=tag)
    elif key.startswith("attr."):
        np.testing.assert_allclose(g, w, rtol=1e-12, atol=0, err_msg=tag)
    elif v in ("k", "r", "mu"):
        np.testing.assert_allclose(g, w, rtol=1e-12, atol=1e-13 if v == "mu" else 0, equal_nan=True, err_msg=tag)
    else:
        assert np.array_equal(np.isnan(g), np.isnan(w)), tag + ": empty bins differ"
        group = key.split(".")[0]
        tol = TOL_F4 if group.replace("-poles", "") in F4_STATS else TOL_F8
        scale = np.nanmax(np.abs(w)) if scale is None else scale
        # ConvolvedFFTPower returns complex64: each side is one rounding (2^-24 relative per part) of an f8 result
        rtol = 2.0 ** -23 if w.dtype == np.complex64 else 0.0
        np.testing.assert_allclose(np.nan_to_num(g), np.nan_to_num(w), rtol=rtol, atol=tol * scale, err_msg=tag)


def _merged(parts):
    """rank 0's result, with the x slabs of the real fields joined"""
    got = dict(parts[0])
    for key in got:
        if key.startswith("field."):
            got[key] = np.concatenate([p[key] for p in parts])
    return got


def _oracle_checks(got, cats, nbar, P0, N, L):
    """the P-rank results against the float64 restatements, at the tolerances of the one-GPU tests"""
    N, L = np.asarray(N), np.asarray(L, dtype="f8")
    V, dk = float(L.prod()), _dk(L)
    p1, w1 = cats["d1"]["Position"], cats["d1"]["Weight"]
    p2 = cats["d2"]["Position"]

    # the window compensation runs in f8 circular coordinates, as nbk_compensate is pinned (test_gpu_mesh_layouts.py,
    # test_gpu_meshapi.py); the reference forms the sinc^3 of interlaced TSC from float32 coordinates, which moves the
    # l = 4 multipole by ~3e-7 of the monopole -- more than the f8 bound below
    wc = po.k_coords(N, L, "f8", kind="circular")

    # FFTPower auto (test_gpu_fftpower.test_mesh_variants_2d_poles)
    real, attrs = po.paint_field(p1, N, L, "tsc", interlaced=True, weight=w1, dtype="f8")
    o = po.power_from_complex(po.compensate("CompensateTSC", wc, po.r2c(real)), None, N, L, mode="2d", Nmu=NMU,
                              poles=POLES, dk=dk, attrs=attrs)
    assert np.array_equal(got["auto.modes"], o["modes"]) and np.array_equal(got["auto-poles.modes"], o["poles_modes"])
    np.testing.assert_allclose(got["auto.k"], o["k"], rtol=1e-5, equal_nan=True)
    np.testing.assert_allclose(got["auto.mu"], o["mu"], rtol=1e-5, atol=1e-7, equal_nan=True)
    atol = 1e-7 * np.nanmax(np.abs(o["poles_power"][0]))
    np.testing.assert_allclose(np.nan_to_num(got["auto.power"].real), np.nan_to_num(o["power"].real), rtol=1e-5, atol=atol)
    for i, ell in enumerate(POLES):
        np.testing.assert_allclose(np.nan_to_num(got["auto-poles.power_%d" % ell].real),
                                   np.nan_to_num(o["poles_power"][i].real), rtol=1e-5, atol=atol, err_msg="auto %d" % ell)
    np.testing.assert_allclose(got["attr.auto.shotnoise"], o["attrs"]["shotnoise"], rtol=1e-12)
    assert got["attr.auto.N1"] == len(p1) and got["attr.auto.N2"] == len(p1)

    def compensated(pos, weight, dtype):
        real, _ = po.paint_field(pos, N, L, "cic", weight=weight, dtype=dtype)
        c = po.r2c(real)
        return po.compensate("CompensateCICShotnoise", wc, c).astype(c.dtype)
    c1 = {t: compensated(p1, w1, t) for t in ("f4", "f8")}
    c2 = {t: compensated(p2, None, t) for t in ("f4", "f8")}

    # FFTPower cross, f4 x f8 (test_gpu_fftpower: f4 meshes to 1e-5 of the monopole)
    for name, los, (t1, t2) in (("cross-x", [1, 0, 0], ("f4", "f8")), ("cross-y", [0, 1, 0], ("f8", "f4"))):
        o = po.power_from_complex(c1[t1], c2[t2], N, L, mode="2d", los=los, Nmu=NMU, poles=[0, 2], dk=dk)
        assert np.array_equal(got[name + ".modes"], o["modes"]), name
        assert np.array_equal(got[name + "-poles.modes"], o["poles_modes"]), name
        np.testing.assert_allclose(got[name + ".k"], o["k"], rtol=1e-5, equal_nan=True)
        atol = 1e-5 * np.nanmax(np.abs(o["poles_power"][0]))
        np.testing.assert_allclose(np.nan_to_num(got[name + ".power"]), np.nan_to_num(o["power"]), rtol=1e-5, atol=atol,
                                   err_msg=name)
        for i, ell in enumerate([0, 2]):
            np.testing.assert_allclose(np.nan_to_num(got[name + "-poles.power_%d" % ell]),
                                       np.nan_to_num(o["poles_power"][i]), rtol=1e-5, atol=atol, err_msg=name)
        assert got["attr.%s.shotnoise" % name] == 0 and got["attr.%s.N2" % name] == len(p2)

    # dk = 0 on the edges the run found (test_gpu_meshapi.test_dk0_at_scale_global_edges)
    p3d = c1["f8"] * np.conj(c1["f8"])
    p3d[0, 0, 0] = 0
    p3d = p3d * V
    res, _ = po.project_to_basis(p3d, po.k_coords(N, L, "f4"), [got["dk0.edges_k"], np.linspace(-1, 1, 2)])
    assert np.array_equal(got["dk0.modes"], np.squeeze(res[3]))
    np.testing.assert_allclose(got["dk0.power"].real, np.squeeze(res[2]).real, rtol=1e-5,
                               atol=1e-8 * np.nanmax(np.abs(res[2])))

    # FFTCorr (test_gpu_meshapi.test_fftcorr_vs_oracle, test_fftcorr_unique_and_padding)
    xi = po.c2r(p3d, N) / V
    xc = co.x_coords(N, L, "f4")
    dr = L.min() / N.max()
    redges = np.arange(0., 0.5 * L.min() + dr / 2, dr)
    res, pres = po.project_to_basis(xi, xc, [redges, np.linspace(0, 1, NMU + 1)], poles=[0, 2], hermitian_symmetric=False)
    assert np.array_equal(got["corr2d.modes"], np.squeeze(res[3]))
    scale = np.nanmax(np.abs(res[2]))
    np.testing.assert_allclose(np.nan_to_num(got["corr2d.corr"]), np.nan_to_num(np.squeeze(res[2]).real), rtol=1e-6,
                               atol=1e-7 * scale)
    np.testing.assert_allclose(got["corr2d.r"], np.squeeze(res[0]), rtol=1e-6, equal_nan=True)
    np.testing.assert_allclose(np.nan_to_num(got["corr2d-poles.corr_2"]), np.nan_to_num(pres[1][1].real), rtol=1e-6,
                               atol=1e-7 * scale)
    assert got["attr.corr2d.N1"] == len(p1)
    res, _ = po.project_to_basis(xi, xc, [got["corr-dr0.edges_r"], np.linspace(0, 1, 2)], hermitian_symmetric=False)
    assert np.array_equal(got["corr-dr0.modes"], np.squeeze(res[3]))
    np.testing.assert_allclose(got["corr-dr0.corr"], np.squeeze(res[2]).real, rtol=1e-6,
                               atol=1e-7 * np.nanmax(np.abs(res[2])))

    # ProjectedFFTPower (test_gpu_meshapi.test_projected_fftpower_reference_assertions)
    real = po.c2r(c1["f8"], N)
    for tag, axes in (("1", [1]), ("01", [0, 1])):
        r = real.sum(axis=tuple(a for a in range(3) if a not in axes))
        cp = np.fft.rfftn(r) / N.prod()
        pk = (cp * cp.conj()).real
        pk.flat[0] = 0
        k = []
        for d, a in enumerate(axes):
            kd = np.fft.fftfreq(N[a], 1. / (N[a] * 2 * np.pi / L[a]))[:pk.shape[d]]
            sh = [1] * len(axes)
            sh[d] = -1
            k.append(kd.reshape(sh))
        kmag = sum(ki ** 2 for ki in k) ** 0.5
        W = np.full(pk.shape, 2.0)
        W[..., 0] = 1.0
        W[..., -1] = 1.0
        edges = got["proj%s.edges_k" % tag]
        dig = np.digitize(kmag.flat, edges)
        nb = len(edges) + 1
        with np.errstate(invalid="ignore", divide="ignore"):
            want = (np.bincount(dig, weights=(W * pk).flat, minlength=nb) /
                    np.bincount(dig, weights=W.flat, minlength=nb))[1:-1] * L[axes].prod()
        assert np.array_equal(got["proj%s.modes" % tag], np.bincount(dig, weights=W.flat, minlength=nb)[1:-1]), tag
        np.testing.assert_allclose(np.nan_to_num(got["proj%s.power" % tag].real), np.nan_to_num(want), rtol=1e-6,
                                   atol=1e-9 * np.nanmax(want), err_msg="projected %s" % tag)

    # MultipleSpeciesCatalog (test_gpu_convpower.test_multiple_species_paint_is_sum_of_single_paints)
    Wa, Wb = float(w1.sum()), float(len(p2))
    npc = (Wa + Wb) / N.prod()
    want = (po.paint(p1, w1, N, L, "cic") + po.paint(p2, None, N, L, "cic")) / npc
    np.testing.assert_allclose(got["field.species"], want, rtol=0, atol=1e-5)
    assert got["attr.species.N"] == len(p1) + len(p2)
    np.testing.assert_allclose([got["attr.species.a.W"], got["attr.species.b.W"], got["attr.species.num_per_cell"]],
                               [Wa, Wb, npc], rtol=1e-12)
    shot = (Wa / (Wa + Wb)) ** 2 * V * float((w1 ** 2).sum()) / Wa ** 2 + (Wb / (Wa + Wb)) ** 2 * V / Wb
    np.testing.assert_allclose(got["attr.species.shotnoise"], shot, rtol=1e-12)

    # ConvolvedFFTPower (test_gpu_convpower.test_convolved_power_vs_oracle, ..._complex_mesh_odd_multipoles)
    fd, fr = cats["fd"], cats["fr"]
    wf = 1. / (1 + P0 * nbar)
    args = (fd["Position"], fr["Position"], (fd["Weight"], wf * np.ones(len(fd["NZ"]))),
            (np.ones(len(fr["NZ"])), wf * np.ones(len(fr["NZ"]))), fd["NZ"], fr["NZ"], N, L)
    pr = fr["Position"]
    centre = 0.5 * (pr.min(axis=0) + pr.max(axis=0))
    for name in ("conv-c16", "conv-f8", "conv-cross"):
        np.testing.assert_array_equal(got["attr.%s.BoxCenter" % name], centre)
    ofull = co.convpower_full(*args, centre, CONV_POLES, resampler="cic", dk=dk)
    o8 = co.convpower(*args, centre, CONV_POLES, resampler="tsc", dk=dk)
    for name, o in (("conv-c16", ofull), ("conv-f8", o8)):
        assert np.array_equal(got[name + ".modes"], o["modes"]), name
        np.testing.assert_allclose(got[name + ".k"], o["k"], rtol=1e-6, equal_nan=True)
        scale = np.nanmax(np.abs(o["power_0"]))
        for ell in CONV_POLES:
            g, w = got["%s.power_%d" % (name, ell)], o["power_%d" % ell]
            for part in ("real", "imag"):
                np.testing.assert_allclose(np.nan_to_num(getattr(g, part)), np.nan_to_num(getattr(w, part)), rtol=1e-5,
                                           atol=2e-6 * scale, err_msg="%s ell %d %s" % (name, ell, part))
        np.testing.assert_allclose(got["attr.%s.alpha" % name], o["alpha"], rtol=1e-12)
    for key, okey in (("alpha", "alpha"), ("data.norm", "data_norm"), ("randoms.norm", "randoms_norm"),
                      ("shotnoise", "shotnoise")):
        for name in ("conv-c16", "conv-f8"):
            np.testing.assert_allclose(got["attr.%s.%s" % (name, key)], o8[okey], rtol=1e-12, err_msg=name + " " + key)


def _problem(gid):
    """the catalogues of geometry `gid`, who holds which row, n(z) and the FKP P0"""
    N, L, P, split = GEOMS[gid]
    cats, nbar = _catalogues(N, L)
    owner = _owners(cats, N, L, P, split)
    if split == "empty":
        assert not any((o == 0).any() for o in owner.values())
    return cats, owner, nbar, 1. / nbar


def _check_ranks(gid, one, parts):
    """the P-rank results (one dict per rank) against one rank's; returns rank 0's with the real-field slabs joined"""
    P = GEOMS[gid][2]
    for r, part in enumerate(parts):
        part = dict(part)
        assert part.pop("c16-raises"), "rank %d: FFTPower on a 'c16' ParticleMesh did not raise on %d ranks" % (r, P)
        assert sorted(part) == sorted(one)
    got = _merged(parts)
    for key in sorted(one):
        scale = _stat_scale(one, key) if _is_stat(key) else None
        if key.startswith("field."):
            _vs_one(got[key], one[key], key, gid)
        else:
            for r, part in enumerate(parts):
                _vs_one(part[key], one[key], key, "%s rank %d" % (gid, r), scale)
    # preview on P ranks is the same run's joined slabs, summed over the dropped axes
    field = got["field.tsc"]
    for tag, want in (("0", field.sum(axis=(1, 2))), ("2", field.sum(axis=(0, 1))), ("20", field.sum(axis=1).T),
                      ("all", field)):
        for r, part in enumerate(parts):
            g = part["preview%s.value" % tag]
            assert g.shape == want.shape, "preview %s rank %d" % (tag, r)
            np.testing.assert_allclose(g, want, rtol=0, atol=1e-12 * np.abs(want).max(), err_msg="preview %s" % tag)
    return got


@pytest.mark.parametrize("gid", sorted(GEOMS))
def test_statistics_on_ranks(cuda, gid):
    """every statistic on P gloo ranks equals one rank (mode counts bit for bit, means to 1e-12, statistics to the
    paint bound, attrs to 1e-12) and the float64 oracle"""
    from nbodykit_b200.comm import SelfComm
    N, L, P, _ = GEOMS[gid]
    cats, owner, nbar, P0 = _problem(gid)
    one = _statistics(SelfComm(), gid, cats, owner, P0)
    parts = _spawn(_statistics, P, gid, cats, owner, P0)
    got = _check_ranks(gid, one, parts)
    _oracle_checks(got, cats, nbar, P0, N, L)


# ---------------------------------------------------------------------------------------------
# B. kernel level on virtual ranks
# ---------------------------------------------------------------------------------------------
# id: (N, dtype, los, Nmu, poles); z is the SYM line of sight, the others the general instance
REAL_BIN_CASES = {"z-odd-f8": ((45, 21, 35), "f8", (0., 0., 1.), 4, [0, 2, 4]),
                  "z-f4": ((48, 36, 17), "f4", (0., 0., 1.), 3, [0, 2]),
                  "oblique-f4": ((30, 33, 16), "f4", (0.6, 0., 0.8), 4, [0, 2, 4]),
                  "oblique-f8": ((48, 36, 17), "f8", (0.6, 0., 0.8), 5, [0, 2, 4]),
                  "y-f8-pow2": ((32, 32, 32), "f8", (0., 1., 0.), 4, [0, 2])}


def _real_bin(t, N, dtype, start, count, edges, los, ells):
    """nbk_power_bin of a real statistic on x planes [start, start + count) as FFTCorr calls it (real_input = 1,
    is_p3d = 1, hermitian = 0, coordinates index x L/N, float32 coordinate mode) -> host raw sums"""
    import torch
    _l = _lib()
    redges, muedges = edges
    Nx, Nmu = len(redges) - 1, len(muedges) - 1
    nb = (Nx + 2) * (Nmu + 2)
    nsum = torch.zeros(nb, dtype=torch.int64, device="cuda")
    xsum = torch.zeros(nb, dtype=torch.float64, device="cuda")
    musum = torch.zeros(nb, dtype=torch.float64, device="cuda")
    ysum = torch.zeros(len(ells) * nb * 2, dtype=torch.float64, device="cuda")
    _l.check(_l.lib().nbk_power_bin(_p(t), None, _code(dtype), 1, 1.0, 1, _l.iarr(N), _l.darr(BOX), 0, start, count, 4,
                                    _l.darr(np.asarray(redges) ** 2), Nx, _l.darr(muedges), Nmu, _l.darr(los),
                                    _l.i32arr(ells), len(ells), 0, 0, 0, 1, _l.darr(np.asarray(BOX) / np.asarray(N)),
                                    _p(nsum), _p(xsum), _p(musum), _p(ysum), None), "nbk_power_bin")
    y = _host(ysum).reshape(len(ells), nb, 2)
    return _host(nsum), _host(xsum), _host(musum), y[..., 0] + 1j * y[..., 1]


@pytest.mark.parametrize("cid", sorted(REAL_BIN_CASES))
def test_real_power_bin_x_slabs(cuda, cid):
    """per-rank sums over x slabs [x_n][Ny][Nz] (layout 0, start = r x_n), summed over the ranks, against
    project_sums(hermitian_symmetric=False) on the wrapped separations of co.x_coords"""
    N, dtype, los, Nmu, poles = REAL_BIN_CASES[cid]
    y = np.random.RandomState(91).standard_normal(N).astype(dtype)
    dr = min(BOX) / max(N)
    edges = (np.arange(0., 0.5 * min(BOX) + dr / 2, dr), np.linspace(0, 1, Nmu + 1))
    ells = [0] + sorted(poles) if 0 not in poles else sorted(poles)
    ref = po.project_sums(y, co.x_coords(N, BOX, "f4"), edges, list(los), poles, hermitian_symmetric=False)
    want = (ref[3], ref[0], ref[1], ref[2])
    tol = 1e-12 if dtype == "f8" else 2e-6
    one = None
    for P in [1] + ml.rank_counts(N[0]):
        x_n = N[0] // P
        tot = None
        for r, s in enumerate(ml.split_x(y, P)):
            got = _real_bin(_dev(s), N, dtype, r * x_n, x_n, edges, los, ells)
            tot = got if tot is None else tuple(a + b for a, b in zip(tot, got))
        _check_sums(tot, want, tol, "%s P=%d vs project_sums" % (cid, P))
        if one is None:
            one = tot
        else:
            _check_sums(tot, one, 1e-13, "%s P=%d vs P=1" % (cid, P))


@pytest.mark.parametrize("N", SIDES)
@pytest.mark.parametrize("dtype", ["f8", "f4"])
@pytest.mark.parametrize("auto", [False, True], ids=["cross", "auto"])
def test_cross_power_transposed_slabs(cuda, N, dtype, auto):
    """c1 conj(c2) V on transposed y slabs with clear_first = (y_start == 0), as fftcorr.py passes it: reassembled, the
    product with only the k = 0 mode cleared -- no rank with y_start > 0 clears its first element"""
    import torch
    _l = _lib()
    rng = np.random.RandomState(81)
    c1, _ = ml.spectra(N, rng, dtype)
    c2 = c1 if auto else ml.spectra(N, rng, dtype)[0]
    V = float(np.prod(BOX))
    want = c1.astype("c16") * np.conj(c2.astype("c16")) * V
    want[0, 0, 0] = 0
    # each part is (a c + b d) V with a product, a sum (possibly fused) and the scale rounded in the field's dtype
    bound = 4 * np.finfo(dtype).eps * np.abs(c1.astype("c16")) * np.abs(c2.astype("c16")) * V
    for P in [1] + ml.rank_counts(N[1]):
        y_n = N[1] // P
        parts = []
        for r, (a, b) in enumerate(zip(ml.split_transposed(c1, P), ml.split_transposed(c2, P))):
            ta = _dev(a)
            tb = None if auto else _dev(b)
            out = torch.empty_like(ta)
            _l.check(_l.lib().nbk_cross_power(_p(ta), _p(tb), _p(out), _code(dtype), out.numel(), V,
                                              1 if r * y_n == 0 else 0, None), "nbk_cross_power")
            parts.append(_host(out))
        got = ml.join_transposed(parts)
        assert got[0, 0, 0] == 0, "P=%d: the k = 0 mode is not cleared" % P
        for r in range(1, P):
            assert got[0, r * y_n, 0] != 0, "P=%d: rank %d (y_start %d) cleared its first element" % (P, r, r * y_n)
        err = np.abs(got - want)
        assert (err <= bound).all(), "P=%d: worst %g over the bound" % (P, (err - bound).max())
