"""ConvolvedFFTBispectrum on the GPU against the float64 oracle (tests/convbispectrum_oracle.py): f8 and f4, CIC and
interlaced TSC on power-of-two, mixed-radix and Bluestein meshes; the exact shot noise of two objects; the far-field
limit against FFTBispectrum; 'c16' against 'f8'; the blocked paths; P = 2, 3 ranks sharing one GPU against one rank.
tests/mgpu_check_convbispectrum.py runs the several-GPU comparison under torchrun.

Tolerances: triangle counts are integers and must match exactly; |dB_ell| <= tol * bound_ell with bound_ell =
V^3 sum |W_a||I_b||I_c| / (I33 sum J J J), and |d shotnoise_0| <= tol * the oracle's shot bound, tol = 1e-10 (f8) or
1e-4 (f4); the norms and S3 to rtol 1e-12."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import convbispectrum_oracle as cbo
from test_gpu_bispectrum import SHAPES, TOL

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLES = [0, 2, 4]
NBAR = 1e-3
COMP = {("cic", False): "CompensateCICShotnoise", ("tsc", True): "CompensateTSC", ("nnb", False): None}


def _columns(L, C, seed, nd=600, nr=3000):
    """data and randoms (10x fewer data) inside the box of side L centred on C, as dicts of numpy columns"""
    rng = np.random.RandomState(seed)
    L, C = np.asarray(L, dtype="f8"), np.asarray(C, dtype="f8")
    cats = {}
    for name, n in (("data", nd), ("randoms", nr)):
        cats[name] = dict(Position=(rng.uniform(-0.45, 0.45, (n, 3)) * L + C),
                          Weight=rng.uniform(0.8, 1.2, n) if name == "data" else np.ones(n),
                          FKPWeight=rng.uniform(0.5, 1.0, n),
                          NZ=np.full(n, NBAR))
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


def _run(cats, N, L, C, dtype="f8", resampler="cic", interlaced=False, comm=None, owner=None, **kw):
    from nbodykit_b200.lab import ConvolvedFFTBispectrum
    mesh = _fkp(cats, comm, owner).to_mesh(Nmesh=N, BoxSize=L, BoxCenter=C, dtype=dtype, resampler=resampler,
                                           interlaced=interlaced)
    return ConvolvedFFTBispectrum(mesh, **kw)


def _want(r, poles, comp, fft=True):
    """the oracle on the fields the call painted (downloaded from its mesh)"""
    mesh = r.first
    F = mesh.compute(mode="real").numpy()
    Nf = mesh.to_shot_field().numpy() if 0 in poles else None
    form = cbo.fft_form if fft else cbo.direct_form
    I33 = r.attrs["randoms.norm3"] or 1.0
    return form(F, Nf, r.attrs["Nmesh"], r.attrs["BoxSize"], r.attrs["BoxCenter"], r.edges, poles, comp, I33,
                r.attrs["S3"])


def _check(r, want, poles, tol, what):
    rows = want["rows"]
    a, b, c = rows.T
    T = want["row_triangles"]
    np.testing.assert_array_equal(r.poles["triangles"][a, b, c], T, err_msg=what)
    ok = T > 0
    assert ok.sum() > 0, what
    for ell in poles:
        B = r.poles["B_%d" % ell][a, b, c]
        assert np.isnan(B[~ok]).all(), what
        err = np.abs(B[ok] - want["B_%d" % ell][ok])
        worst = (err / want["bound_%d" % ell][ok]).max()
        assert (err <= tol * want["bound_%d" % ell][ok]).all(), "%s ell=%d: |dB| / bound = %.3g" % (what, ell, worst)
    if 0 in poles:
        i, j, l = want["triples"].T
        okt = want["triangles"] > 0
        sn = r.poles["shotnoise_0"][i, j, l]
        assert np.isnan(sn[~okt]).all(), what
        err = np.abs(sn[okt] - want["shotnoise_0"][okt])
        assert (err <= tol * want["shot_bound"][okt]).all(), "%s shot: %.3g" % (
            what, (err / want["shot_bound"][okt]).max())


def _geom(shape):
    N, L = SHAPES[shape]
    C = np.array([350., -820., 1240.])          # an off-origin survey volume
    return N, np.asarray(L), C


@pytest.mark.parametrize("window", [("cic", False), ("tsc", True)])
@pytest.mark.parametrize("dtype", ["f8", "f4"])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_matches_oracle(cuda, shape, dtype, window):
    N, L, C = _geom(shape)
    cats = _columns(L, C, 31)
    r = _run(cats, N, L, C, dtype, *window, poles=POLES)
    want = _want(r, POLES, COMP[window])
    _check(r, want, POLES, TOL[dtype], "%s %s %s" % (shape, dtype, window))
    p = r.poles
    assert p.dims == ["k1", "k2", "k3"]
    assert p.data.dtype.names == ("k1", "k2", "k3", "B_0", "B_2", "B_4", "shotnoise_0", "triangles")
    B0 = p["B_0"]
    for perm in ((0, 2, 1), (1, 0, 2), (2, 1, 0)):
        np.testing.assert_array_equal(np.isnan(B0), np.isnan(np.transpose(B0, perm)))
        np.testing.assert_array_equal(np.nan_to_num(B0), np.nan_to_num(np.transpose(B0, perm)))
    for ell in (2, 4):
        B = p["B_%d" % ell]
        np.testing.assert_array_equal(np.nan_to_num(B), np.nan_to_num(np.transpose(B, (0, 2, 1))))
    # the norms and S3 from the catalogue columns
    d, rr = cats["data"], cats["randoms"]
    alpha = d["Weight"].sum() / rr["Weight"].sum()
    np.testing.assert_allclose(r.attrs["alpha"], alpha, rtol=1e-12)
    np.testing.assert_allclose(r.attrs["data.norm3"], (NBAR ** 2 * d["Weight"] * d["FKPWeight"] ** 3).sum(), rtol=1e-12)
    np.testing.assert_allclose(r.attrs["randoms.norm3"],
                               alpha * (NBAR ** 2 * rr["Weight"] * rr["FKPWeight"] ** 3).sum(), rtol=1e-12)
    S3 = ((d["Weight"] * d["FKPWeight"]) ** 3).sum() - alpha ** 3 * ((rr["Weight"] * rr["FKPWeight"]) ** 3).sum()
    np.testing.assert_allclose(r.attrs["S3"], S3, rtol=1e-12)
    nshell = len(r.edges) - 1
    assert r.attrs["transforms"] == 1 + 5 + 9 + 1 + (3 + 2) * nshell
    for key in ("data.N", "randoms.N", "data.W", "randoms.W"):
        assert key in r.attrs


def test_fields_are_the_oracle_paint(cuda):
    """F and the shot field N of a CIC f8 mesh are convpower_oracle.fkp_field's paint (mass u, and u^2 with +alpha^2)"""
    N, L, C = _geom("48x36x30")
    cats = _columns(L, C, 32)
    r = _run(cats, N, L, C, "f8", "cic", poles=[0])
    d, rr = cats["data"], cats["randoms"]
    cols = lambda c: dict(wc=c["Weight"], wf=c["FKPWeight"], nbar=c["NZ"], v=np.ones(len(c["NZ"])))   # noqa: E731
    f = cbo.fkp_fields(d["Position"], rr["Position"], cols(d), cols(rr), N, L, C, "cic")
    scale = np.abs(f["F"]).max()
    np.testing.assert_allclose(r.first.compute(mode="real").numpy(), f["F"], rtol=0, atol=1e-11 * scale)
    np.testing.assert_allclose(r.first.to_shot_field().numpy(), f["N"], rtol=0, atol=1e-11 * np.abs(f["N"]).max())
    for key, name in (("data.norm3", "data_norm3"), ("randoms.norm3", "randoms_norm3"), ("S3", "S3"),
                      ("alpha", "alpha")):
        np.testing.assert_allclose(r.attrs[key], f[name], rtol=1e-12)


def test_direct_sum_16(cuda):
    """independent of every FFT and of Y_lm: the oracle's direct sum over closed triangles at 16 x 12 x 10"""
    N, L, C = (16, 12, 10), np.array([160., 120., 100.]), np.array([-40., 900., 300.])
    cats = _columns(L, C, 33, nd=300, nr=1500)
    r = _run(cats, N, L, C, "f8", "cic", poles=POLES)
    want = _want(r, POLES, COMP[("cic", False)], fft=False)
    fft = _want(r, POLES, COMP[("cic", False)])
    for ell in POLES:
        want["bound_%d" % ell] = fft["bound_%d" % ell]
    want["shot_bound"] = fft["shot_bound"]
    _check(r, want, POLES, TOL["f8"], "direct 16x12x10")


def test_exact_shot_noise_of_two_objects(cuda):
    """one data and one random object on distinct grid nodes, NNB, no compensation, unit weights, equal NZ: every term
    of the raw estimator is a coincidence term, so B_0 = shotnoise_0.  The data object carries Value = 2: with equal
    masses the pair terms are odd in q and both sides vanish identically."""
    N, L, C = (32, 32, 32), np.array([200., 200., 200.]), np.array([1000., -500., 300.])
    H = L / np.array(N)
    cats = {"data": dict(Position=(C + np.array([3, -5, 7]) * H)[None], NZ=np.full(1, NBAR), Value=np.full(1, 2.)),
            "randoms": dict(Position=(C + np.array([-9, 2, 11]) * H)[None], NZ=np.full(1, NBAR), Value=np.ones(1))}
    for c in cats.values():
        c["Weight"] = np.ones(1)
        c["FKPWeight"] = np.ones(1)
    r = _run(cats, N, L, C, "f8", "nnb", poles=[0])
    assert r.attrs["alpha"] == 1.0 and r.attrs["S3"] == 7.0
    B, S, T = r.poles["B_0"], r.poles["shotnoise_0"], r.poles["triangles"]
    ok = T > 0
    assert ok.sum() > 100
    np.testing.assert_array_equal(np.isnan(B), ~ok)
    np.testing.assert_array_equal(np.isnan(S), ~ok)
    assert np.abs(B[ok]).min() > 1e-6 * np.abs(B[ok]).max()
    assert (np.abs(B[ok] - S[ok]) <= 1e-10 * np.abs(B[ok])).all(), (np.abs(B[ok] - S[ok]) / np.abs(B[ok])).max()


def test_far_field_limit(cuda):
    """the survey at BoxCenter = (0, 0, 1e4 L): x_hat is z to 1e-4, so the end-point multipoles are FFTBispectrum's
    about los = z on the same field; B_0 I33 / V is FFTBispectrum's B (the same estimator, uncompensated NNB)"""
    from nbodykit_b200.lab import FFTBispectrum, FieldMesh
    N, L = (32, 32, 32), np.array([200., 200., 200.])
    C = np.array([0., 0., 1e4 * L[2]])
    cats = _columns(L, C, 34)
    r = _run(cats, N, L, C, "f8", "nnb", poles=POLES)
    F = r.first.compute(mode="real")
    ref = FFTBispectrum(FieldMesh(F), poles=POLES, los=[0, 0, 1])
    np.testing.assert_array_equal(ref.poles["triangles"], r.poles["triangles"])
    want = _want(r, POLES, None)
    a, b, c = want["rows"].T
    ok = want["row_triangles"] > 0
    I33, V = r.attrs["randoms.norm3"], float(np.prod(L))
    err0 = np.abs(r.poles["B_0"][a, b, c] * I33 / V - ref.poles["B_0"][a, b, c])[ok]
    assert (err0 <= 1e-10 * want["bound_0"][ok] * I33 / V).all()
    for ell in (2, 4):
        err = np.abs(r.poles["B_%d" % ell][a, b, c] * I33 / V - ref.poles["B_%d" % ell][a, b, c])[ok]
        assert (err <= 1e-3 * want["bound_%d" % ell][ok] * I33 / V).all(), (ell, (err / want["bound_%d" % ell][ok]
                                                                                   / I33 * V).max())


def test_complex_mesh_equals_real(cuda):
    N, L, C = _geom("48x36x30")
    cats = _columns(L, C, 35)
    r8 = _run(cats, N, L, C, "f8", "tsc", True, poles=POLES)
    r16 = _run(cats, N, L, C, "c16", "tsc", True, poles=POLES)
    want = _want(r8, POLES, COMP[("tsc", True)])
    _check(r16, want, POLES, TOL["f8"], "c16")
    np.testing.assert_array_equal(r16.poles["triangles"], r8.poles["triangles"])


@pytest.mark.parametrize("cap", [3, 4, 20])
def test_blocked_path_matches_resident(cuda, monkeypatch, cap):
    """NBK_BISPEC_RESIDENT = 3, 4: shell blocks per family in both passes; 20 (8 shells: the I pass one family at a
    time, the J pass with its H family resident)"""
    N, L, C = _geom("32")
    cats = _columns(L, C, 36)
    kw = dict(dk=2 * 2 * np.pi / L[0], poles=POLES)
    one = _run(cats, N, L, C, "f8", "cic", **kw)
    nshell = len(one.edges) - 1
    assert nshell == 8 and one.attrs["transforms"] == 16 + 5 * nshell
    monkeypatch.setenv("NBK_BISPEC_RESIDENT", str(cap))
    blk = _run(cats, N, L, C, "f8", "cic", **kw)
    if cap == 20:
        assert blk.attrs["transforms"] == 16 + 5 * nshell
    else:
        assert blk.attrs["transforms"] > 16 + 5 * nshell
    want = _want(one, POLES, COMP[("cic", False)])
    np.testing.assert_array_equal(blk.poles["triangles"], one.poles["triangles"])
    a, b, c = want["rows"].T
    ok = want["row_triangles"] > 0
    for ell in POLES:
        err = np.abs(blk.poles["B_%d" % ell] - one.poles["B_%d" % ell])[a, b, c][ok]
        assert (err <= 1e-12 * want["bound_%d" % ell][ok]).all(), (cap, ell)
    i, j, l = want["triples"].T
    okt = want["triangles"] > 0
    err = np.abs(blk.poles["shotnoise_0"] - one.poles["shotnoise_0"])[i, j, l][okt]
    assert (err <= 1e-12 * want["shot_bound"][okt]).all(), cap


def _on_ranks(comm, shape, cats, owner):
    N, L, C = _geom(shape)
    r = _run(cats, N, L, C, "f8", "tsc", True, comm=comm, owner=owner, poles=POLES)
    return dict(poles={f: r.poles[f] for f in r.poles.data.dtype.names}, attrs={k: r.attrs[k] for k in
                                                                                ("data.norm3", "randoms.norm3", "S3")})


@pytest.mark.parametrize("shape,P", [("32", 2), ("48x36x30", 3)])
def test_ranks_match_one(cuda, shape, P):
    from test_gpu_slab_route import _spawn
    N, L, C = _geom(shape)
    cats = _columns(L, C, 37)
    rng = np.random.RandomState(3)
    owner = {name: rng.randint(0, P, len(c["NZ"])) for name, c in cats.items()}
    one = _run(cats, N, L, C, "f8", "tsc", True, poles=POLES)
    want = _want(one, POLES, COMP[("tsc", True)])
    parts = _spawn(_on_ranks, P, shape, cats, owner)
    a, b, c = want["rows"].T
    ok = want["row_triangles"] > 0
    i, j, l = want["triples"].T
    okt = want["triangles"] > 0
    for rank, part in enumerate(parts):
        np.testing.assert_array_equal(part["poles"]["triangles"], one.poles["triangles"])
        for ell in POLES:
            err = np.abs(part["poles"]["B_%d" % ell] - one.poles["B_%d" % ell])[a, b, c][ok]
            assert (err <= 1e-10 * want["bound_%d" % ell][ok]).all(), (shape, rank, ell)
        err = np.abs(part["poles"]["shotnoise_0"] - one.poles["shotnoise_0"])[i, j, l][okt]
        assert (err <= 1e-10 * want["shot_bound"][okt]).all(), (shape, rank)
        for k, v in part["attrs"].items():
            np.testing.assert_allclose(v, one.attrs[k], rtol=1e-12)


def test_two_gpu_convbispectrum_matches_one_gpu():
    """launches tests/mgpu_check_convbispectrum.py under torchrun when the box has >= 2 GPUs"""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29547", os.path.join(ROOT, "tests", "mgpu_check_convbispectrum.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    sys.stdout.write(out.stdout[-3000:])
    sys.stderr.write(out.stderr[-3000:])
    assert out.returncode == 0
