"""FFTBispectrum multipoles (poles=, los=) on the GPU against the float64 oracle (tests/bispectrum_poles_oracle.py): the
FFT form on power-of-two, mixed-radix and Bluestein meshes in f4 and f8 with three lines of sight, the FFT-free direct
sum at 16^3, B_0 against .bispec, the quadrupole sum rule over the three axes, plane waves in closed form, the blocked
and one-family-at-a-time paths, and P = 2, 3, 4 ranks sharing one GPU against one rank.
tests/mgpu_check_bispectrum_poles.py runs the several-GPU comparison under torchrun.

Tolerances: triangle counts are integers and must match exactly; |dB_ell| <= tol * bound_ell with
bound_ell = (2 ell + 1) V^2 sum |W_a||I_b||I_c| / sum J J J (the oracle's), tol = 1e-10 (f8) or 1e-4 (f4)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import bispectrum_poles_oracle as bpo
from test_gpu_bispectrum import SHAPES, TOL, _field, _half, _mesh

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLES = [0, 2, 4]
LOS = {"z": [0, 0, 1], "x": [1, 0, 0], "diag": list(np.ones(3) / np.sqrt(3))}


def _run(mesh, **kw):
    from nbodykit_b200.lab import FFTBispectrum
    return FFTBispectrum(mesh, **kw)


def _rows(r, rows, ell):
    a, b, c = np.asarray(rows).T
    return r.poles["B_%d" % ell][a, b, c], r.poles["triangles"][a, b, c]


def _check(r, want, tol, what):
    for ell, w in want.items():
        B, T = _rows(r, w["rows"], ell)
        np.testing.assert_array_equal(T, w["triangles"], err_msg="%s ell=%d" % (what, ell))
        ok = w["triangles"] > 0
        assert ok.sum() > 0, what
        assert np.isnan(B[~ok]).all(), what
        err = np.abs(B[ok] - w["B"][ok])
        worst = (err / w["bound"][ok]).max()
        assert (err <= tol * w["bound"][ok]).all(), "%s ell=%d: |dB| / bound = %.3g > %g" % (what, ell, worst, tol)


@pytest.mark.parametrize("los", sorted(LOS))
@pytest.mark.parametrize("dtype", ["f8", "f4"])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_matches_oracle(cuda, shape, dtype, los):
    N, L = SHAPES[shape]
    mesh = _mesh(_field(N, 11), L, dtype)
    r = _run(mesh, poles=POLES, los=LOS[los])
    kedges = r.bispec.edges["k1"]
    nshell = len(kedges) - 1
    want = bpo.fft_form_poles(_half(mesh), N, L, kedges, POLES, LOS[los])
    _check(r, want, TOL[dtype], "%s %s los=%s" % (shape, dtype, los))
    p = r.poles
    assert p.dims == ["k1", "k2", "k3"] and p.data.dtype.names == ("k1", "k2", "k3", "B_0", "B_2", "B_4", "triangles")
    np.testing.assert_array_equal(p["B_0"], r.bispec["B"])
    np.testing.assert_array_equal(p["triangles"], r.bispec["triangles"])
    np.testing.assert_array_equal(p["k1"], r.bispec["k1"])
    for ell in (2, 4):
        B = p["B_%d" % ell]
        np.testing.assert_array_equal(B, np.transpose(B, (0, 2, 1)))
        np.testing.assert_array_equal(np.isnan(B), r.bispec["triangles"] == 0)
    assert 3 * nshell <= 64 and r.attrs["transforms"] == (2 + 2) * nshell
    assert r.attrs["poles"] == POLES and r.attrs["los"] == LOS[los]


def test_b0_and_default_call(cuda):
    """B_0 is the call's .bispec['B'] bit for bit, .bispec does not depend on poles (to the float64 atomics of the
    triple sum, whose order differs from call to call), and a call without poles runs 2 nshell transforms and has no
    .poles"""
    from oracle import bispectrum_oracle as bo
    N, L = SHAPES["48x36x30"]
    mesh = _mesh(_field(N, 12), L, "f8")
    plain = _run(mesh)
    kedges = plain.bispec.edges["k1"]
    nshell = len(kedges) - 1
    assert plain.poles is None and plain.attrs["transforms"] == 2 * nshell and plain.attrs["poles"] == []
    only0 = _run(mesh, poles=[0])
    assert only0.attrs["transforms"] == 2 * nshell
    r = _run(mesh, poles=[2, 0], los=LOS["x"])
    assert r.attrs["transforms"] == 3 * nshell
    want = bo.fft_form(_half(mesh), N, L, kedges)
    i, j, l = want["triples"].T
    ok = want["triangles"] > 0
    for x in (only0, r):
        np.testing.assert_array_equal(x.poles["B_0"], x.bispec["B"])
        np.testing.assert_array_equal(x.bispec["triangles"], plain.bispec["triangles"])
        err = np.abs(x.bispec["B"][i, j, l] - plain.bispec["B"][i, j, l])[ok]
        assert (err <= 1e-13 * want["bound"][ok]).all()
        np.testing.assert_allclose(x.power["power"], plain.power["power"], rtol=1e-12)
    assert r.poles.data.dtype.names == ("k1", "k2", "k3", "B_2", "B_0", "triangles")


def test_direct_sum_16(cuda):
    """independent of every FFT: the direct sum over closed triangles at 16^3"""
    N, L = (16, 16, 16), (100., 100., 100.)
    mesh = _mesh(_field(N, 13), L, "f8")
    r = _run(mesh, poles=POLES, los=LOS["diag"])
    kedges = r.bispec.edges["k1"]
    half = _half(mesh)
    want = bpo.direct_form_poles(half, N, L, kedges, POLES, LOS["diag"])
    fft = bpo.fft_form_poles(half, N, L, kedges, POLES, LOS["diag"])
    for ell in POLES:
        want[ell]["bound"] = fft[ell]["bound"]
    _check(r, want, TOL["f8"], "direct 16^3")


def test_quadrupole_sum_rule(cuda):
    """L_2(qx/q) + L_2(qy/q) + L_2(qz/q) = 0: B_2 with los = x, y and z sums to zero on a cubic mesh (to float32
    rounding of mu)"""
    N, L = SHAPES["32"]
    mesh = _mesh(_field(N, 14), L, "f8")
    half = _half(mesh)
    total, bound = 0., 0.
    tri = None
    for los in ([1, 0, 0], [0, 1, 0], [0, 0, 1]):
        r = _run(mesh, poles=[2], los=los)
        if tri is None:
            tri = r.poles["triangles"]
        np.testing.assert_array_equal(r.poles["triangles"], tri)
        w = bpo.fft_form_poles(half, N, L, r.bispec.edges["k1"], [2], los)[2]
        B, _ = _rows(r, w["rows"], 2)
        ok = w["triangles"] > 0
        total = total + np.where(ok, B, 0.)
        bound = bound + w["bound"]
    assert ok.sum() > 100
    worst = (np.abs(total[ok]) / bound[ok]).max()
    assert (np.abs(total[ok]) <= 1e-6 * bound[ok]).all(), worst


def test_plane_waves_closed_form(cuda):
    """delta = sum_a 2 A cos(q_a.x + phi_a) with q1 = (2, 0, 0) kf, q2 = (0, 3, 0) kf, q3 = -(q1 + q2): only (q1, q2, q3)
    and its mirror carry signal, so B_2[1, 2, 3] T / V^2 = 5 L_2(mu(q1)) 2 A^3 cos(phi1 + phi2 + phi3), and
    B_2[2, 1, 3] weights mu(q2)"""
    N, L = (32, 32, 32), (100., 100., 100.)
    kf = 2 * np.pi / L[0]
    q = np.array([[2, 0, 0], [0, 3, 0], [-2, -3, 0]])
    A, phi = 0.3, [0.3, -0.2, 0.6]
    x = np.indices(N).reshape(3, -1).T * (L[0] / N[0])
    arr = sum(2 * A * np.cos(x @ (qa * kf) + p) for qa, p in zip(q, phi)).reshape(N)
    V = np.prod(L)
    signal = 2 * A ** 3 * np.cos(sum(phi))
    kf32 = np.float32(2 * np.pi / L[0])
    for los, mu1, mu2 in (([1, 0, 0], 1., 0.), ([0, 0, 1], 0., 0.)):
        r = _run(_mesh(arr, L, "f8"), dk=kf, kmin=0.5 * kf, kmax=4.6 * kf, poles=[2], los=los)
        for (a, b, c), qa, mu in (((1, 2, 3), q[0], mu1), ((2, 1, 3), q[1], mu2)):
            m = bpo._mu(*[np.float32(v) * kf32 for v in qa], los)
            assert float(m) == mu
            B = r.poles["B_2"][a, b, c] * r.poles["triangles"][a, b, c] / V ** 2
            want = 5 * bpo.legendre(2, mu) * signal
            assert abs(B - want) <= 1e-10 * A ** 3, (los, (a, b, c), B, want)
            assert r.poles["B_2"][a, c, b] == r.poles["B_2"][a, b, c]


@pytest.mark.parametrize("cap", [3, 4, 20])
def test_blocked_path_matches_resident(cuda, monkeypatch, cap):
    """NBK_BISPEC_RESIDENT = 3, 4: shell blocks per family; 20 (two of the three families of 8 shells): one family at a
    time, every field built once"""
    N, L = SHAPES["32"]
    mesh = _mesh(_field(N, 15), L, "f8")
    kw = dict(dk=2 * 2 * np.pi / L[0], poles=POLES, los=LOS["diag"])
    one = _run(mesh, **kw)
    kedges = one.bispec.edges["k1"]
    nshell = len(kedges) - 1
    assert nshell == 8 and one.attrs["transforms"] == 4 * nshell
    monkeypatch.setenv("NBK_BISPEC_RESIDENT", str(cap))
    blk = _run(mesh, **kw)
    if cap == 20:
        assert blk.attrs["transforms"] == 4 * nshell
    else:
        assert blk.attrs["transforms"] > 4 * nshell
    want = bpo.fft_form_poles(_half(mesh), N, L, kedges, POLES, LOS["diag"])
    np.testing.assert_array_equal(blk.poles["triangles"], one.poles["triangles"])
    for ell in POLES:
        B1, _ = _rows(one, want[ell]["rows"], ell)
        B2, _ = _rows(blk, want[ell]["rows"], ell)
        ok = want[ell]["triangles"] > 0
        assert (np.abs(B2 - B1)[ok] <= 1e-13 * want[ell]["bound"][ok]).all(), (cap, ell)


def _record_passes(cls, setattr_=setattr):
    """replaces cls._pass (through setattr_) by a wrapper that appends (indicator, ells, transforms, peak bytes
    allocated above the pass's start) for every pass to the returned list"""
    orig = cls._pass
    seen = []

    def rec(self, c, kedges, triples, indicator, ells=()):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out = orig(self, c, kedges, triples, indicator, ells)
        torch.cuda.synchronize()
        seen.append((indicator, tuple(ells), out[1], torch.cuda.max_memory_allocated() - base))
        return out
    setattr_(cls, "_pass", rec)
    return seen


@pytest.mark.parametrize("cap", [None, 12, 20])
def test_indicator_pass_is_the_plain_one(cuda, monkeypatch, cap):
    """the J pass of a call with multipoles builds only the J fields: it runs the plain call's transforms and holds
    its peak memory, resident (no cap), with the I pass blocked (nshell <= cap < 2 nshell) and one family at a time
    (cap = 2 nshell + 4)"""
    from nbodykit_b200.algorithms.bispectrum import FFTBispectrum
    N, L = SHAPES["32"]
    mesh = _mesh(_field(N, 18), L, "f8")
    kw = dict(dk=2 * 2 * np.pi / L[0])
    if cap:
        monkeypatch.setenv("NBK_BISPEC_RESIDENT", str(cap))
    seen = _record_passes(FFTBispectrum, monkeypatch.setattr)
    plain = _run(mesh, **kw)
    r = _run(mesh, poles=POLES, los=LOS["diag"], **kw)
    nshell = len(plain.bispec.edges["k1"]) - 1
    assert nshell == 8
    (pi, _, pn, _), (pj, pje, pjn, pjm), (ri, rie, rin, _), (rj, rje, rjn, rjm) = seen
    assert (pi, pj, ri, rj) == (False, True, False, True)
    assert pje == () and rje == () and rie == (2, 4)
    assert pn == pjn == rjn == nshell
    assert rjm <= pjm
    if cap == 12:
        assert rin > 3 * nshell                                      # the I pass takes shell blocks
    else:
        assert rin == 3 * nshell and r.attrs["transforms"] == 4 * nshell
    assert r.attrs["transforms"] == rin + rjn


def _on_ranks(comm, gid, cap):
    from test_gpu_rank_statistics import GEOMS
    N, L, _, _ = GEOMS[gid]
    from nbodykit_b200.algorithms.bispectrum import FFTBispectrum
    if cap:
        os.environ["NBK_BISPEC_RESIDENT"] = str(cap)
    seen = _record_passes(FFTBispectrum)               # this process ends with the call
    r = _run(_mesh(_field(N, 17), L, "f8", comm), poles=POLES, los=LOS["diag"])
    return dict(poles={ell: r.poles["B_%d" % ell] for ell in POLES}, T=r.poles["triangles"],
                transforms=r.attrs["transforms"], j_transforms=[n for ind, _, n, _ in seen if ind])


@pytest.mark.parametrize("gid", ["32-P2", "32-P4", "48x36x30-P3", "44x22x26-P2"])
def test_ranks_match_one(cuda, gid):
    from test_gpu_rank_statistics import GEOMS
    from test_gpu_slab_route import _spawn
    N, L, P, _ = GEOMS[gid]
    mesh = _mesh(_field(N, 17), L, "f8")
    one = _run(mesh, poles=POLES, los=LOS["diag"])
    want = bpo.fft_form_poles(_half(mesh), N, L, one.bispec.edges["k1"], POLES, LOS["diag"])
    cap = 24 if gid == "32-P2" else 0         # one geometry also takes the blocked path (48 fields) on every rank
    parts = _spawn(_on_ranks, P, gid, cap)
    for r, part in enumerate(parts):
        np.testing.assert_array_equal(part["T"], one.poles["triangles"], err_msg="%s rank %d" % (gid, r))
        for ell in POLES:
            a, b, c = want[ell]["rows"].T
            ok = want[ell]["triangles"] > 0
            err = np.abs(part["poles"][ell][a, b, c] - one.poles["B_%d" % ell][a, b, c])[ok]
            assert (err <= 1e-12 * want[ell]["bound"][ok]).all(), "%s rank %d ell %d" % (gid, r, ell)
        # the J pass is never blocked here (nshell <= cap): one transform per shell on every rank
        assert part["j_transforms"] == [len(one.bispec.edges["k1"]) - 1], "%s rank %d" % (gid, r)
        if cap:
            assert part["transforms"] > one.attrs["transforms"]


def test_two_gpu_bispectrum_poles_matches_one_gpu():
    """launches tests/mgpu_check_bispectrum_poles.py under torchrun when the box has >= 2 GPUs"""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29543", os.path.join(ROOT, "tests", "mgpu_check_bispectrum_poles.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    sys.stdout.write(out.stdout[-3000:])
    sys.stderr.write(out.stderr[-3000:])
    assert out.returncode == 0
