"""FFTBispectrum on the GPU against the float64 oracle (oracle/bispectrum_oracle.py): the FFT form on power-of-two,
mixed-radix and Bluestein meshes in f4 and f8, the FFT-free direct sum at 16^3, a plane-wave field whose bispectrum is
known in closed form, the 1-D power against FFTPower, the blocked path, P = 2, 3, 4 ranks sharing one GPU against one
rank, and empty shells.  tests/mgpu_check_bispectrum.py runs the several-GPU comparison under torchrun.

Tolerances: triangle counts are integers and must match exactly; |dB| <= tol * bound with
bound = V^2 sum |I_i||I_j||I_l| / sum J_i J_j J_l (the oracle's), tol = 1e-10 (f8) or 1e-4 (f4)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import bispectrum_oracle as bo

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = {"f8": 1e-10, "f4": 1e-4}
# (Nmesh, BoxSize): power of two, mixed radix on a non-cubic box, Bluestein (11 and 13 are prime)
SHAPES = {"32": ((32, 32, 32), (200., 200., 200.)),
          "48x36x30": ((48, 36, 30), (100., 130., 70.)),
          "44x22x26": ((44, 22, 26), (120., 70., 90.))}


def _field(N, seed):
    """a skewed real field: a Gaussian plus half its square"""
    g = np.random.RandomState(seed).normal(size=N)
    return g + 0.5 * (g ** 2 - 1)


def _mesh(arr, L, dtype, comm=None):
    """FieldMesh of this rank's x slab of the full real array `arr`"""
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import FieldMesh
    from nbodykit_b200.pmesh.pm import ParticleMesh
    comm = comm if comm is not None else SelfComm()
    pm = ParticleMesh(BoxSize=L, Nmesh=arr.shape, dtype=dtype, comm=comm)
    rdt = "f4" if dtype in ("f4", "c8") else "f8"
    slab = np.ascontiguousarray(arr[pm.x_start:pm.x_start + pm.x_n].astype(rdt))
    return FieldMesh(pm.create(type="real", value=slab))


def _run(mesh, **kw):
    from nbodykit_b200.lab import FFTBispectrum
    return FFTBispectrum(mesh, **kw)


def _half(mesh):
    """the compressed spectrum the estimator binned, downloaded (one rank)"""
    c = mesh.compute(mode="complex")
    a = c.numpy()
    return a if c.compressed else a[..., :c.pm.Nmesh[2] // 2 + 1]


def _flat(r, tri):
    """B and triangles of `r.bispec` at the sorted triples"""
    i, j, l = np.asarray(tri).T
    return r.bispec["B"][i, j, l], r.bispec["triangles"][i, j, l]


def _check(r, want, tol, what):
    B, T = _flat(r, want["triples"])
    np.testing.assert_array_equal(T, want["triangles"], err_msg=what)
    ok = want["triangles"] > 0
    assert ok.sum() > 0, what
    assert np.isnan(B[~ok]).all(), what
    err = np.abs(B[ok] - want["B"][ok])
    worst = (err / want["bound"][ok]).max()
    assert (err <= tol * want["bound"][ok]).all(), "%s: |dB| / bound = %.3g > %g" % (what, worst, tol)


@pytest.mark.parametrize("dtype", ["f8", "f4"])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_matches_oracle(cuda, shape, dtype):
    N, L = SHAPES[shape]
    mesh = _mesh(_field(N, 11), L, dtype)
    r = _run(mesh)
    kedges = r.bispec.edges["k1"]
    want = bo.fft_form(_half(mesh), N, L, kedges)
    _check(r, want, TOL[dtype], "%s %s" % (shape, dtype))
    # every permutation of a triple is filled with the same numbers
    d = r.bispec.data
    for perm in [(0, 2, 1), (1, 0, 2), (2, 1, 0)]:
        np.testing.assert_array_equal(np.transpose(d["triangles"], perm), d["triangles"])
        np.testing.assert_array_equal(np.transpose(d["B"], perm), d["B"])
    assert r.attrs["transforms"] == 2 * (len(kedges) - 1)
    for key in ("Nmesh", "BoxSize", "volume", "dk", "kmin", "kmax", "N1", "shotnoise", "transforms"):
        assert key in r.attrs


def test_complex_mesh_is_compressed(cuda):
    """a complex-dtype mesh (full spectrum) gives what the real-dtype mesh gives"""
    N, L = SHAPES["48x36x30"]
    arr = _field(N, 12)
    r8 = _run(_mesh(arr, L, "f8"))
    r16 = _run(_mesh(arr, L, "c16"))
    want = bo.fft_form(_half(_mesh(arr, L, "f8")), N, L, r8.bispec.edges["k1"])
    _check(r16, want, TOL["f8"], "c16")
    np.testing.assert_array_equal(r16.bispec["triangles"], r8.bispec["triangles"])


def test_direct_sum_16(cuda):
    """independent of every FFT: the direct sum over closed triangles at 16^3"""
    N, L = (16, 16, 16), (100., 100., 100.)
    mesh = _mesh(_field(N, 13), L, "f8")
    r = _run(mesh)
    kedges = r.bispec.edges["k1"]
    half = _half(mesh)
    want = bo.direct_form(half, N, L, kedges)
    want["bound"] = bo.fft_form(half, N, L, kedges)["bound"]
    _check(r, want, TOL["f8"], "direct 16^3")


def test_plane_waves_closed_form(cuda):
    """delta = sum_a 2 A cos(q_a.x + phi_a) with q1 + q2 + q3 = 0 in three distinct shells: the only closed triplets
    carrying signal are (q1, q2, q3) and its mirror, so B T / V^2 = 2 A^3 cos(phi1 + phi2 + phi3); phi1 + pi flips it"""
    N, L = (32, 32, 32), (100., 100., 100.)
    kf = 2 * np.pi / L[0]
    q = np.array([[2, 0, 0], [0, 3, 0], [-2, -3, 0]])          # |q| = 2, 3, 3.61 kf
    A = 0.3
    x = np.indices(N).reshape(3, -1).T * (L[0] / N[0])
    out = []
    for phi in ([0.3, -0.2, 0.6], [0.3 + np.pi, -0.2, 0.6]):
        arr = sum(2 * A * np.cos(x @ (qa * kf) + p) for qa, p in zip(q, phi)).reshape(N)
        r = _run(_mesh(arr, L, "f8"), dk=kf, kmin=0.5 * kf, kmax=4.6 * kf)
        V = np.prod(L)
        b = r.bispec["B"][1, 2, 3] * r.bispec["triangles"][1, 2, 3] / V ** 2
        want = 2 * A ** 3 * np.cos(sum(phi))
        assert abs(b - want) <= 1e-10 * A ** 3, (b, want)
        out.append(b)
    assert out[0] * out[1] < 0 and abs(out[0] + out[1]) <= 1e-10 * A ** 3


def test_power_matches_fftpower(cuda):
    from nbodykit_b200.lab import FFTPower
    N, L = SHAPES["48x36x30"]
    mesh = _mesh(_field(N, 14), L, "f8")
    kw = dict(dk=0.03, kmin=0.05, kmax=0.6)
    r = _run(mesh, **kw)
    p = FFTPower(mesh, mode="1d", **kw).power
    np.testing.assert_array_equal(r.power["modes"], p["modes"])
    np.testing.assert_allclose(r.power["power"], p["power"], rtol=1e-12)
    np.testing.assert_allclose(r.power["k"], p["k"], rtol=1e-12)
    # the shells' mean |k| are the FFTPower bins' (k = 0 is below kmin here)
    np.testing.assert_allclose(r.bispec["k1"][:, 0, 0], p["k"], rtol=1e-12)


def test_blocked_path_matches_resident(cuda, monkeypatch):
    N, L = SHAPES["32"]
    mesh = _mesh(_field(N, 15), L, "f8")
    kw = dict(dk=2 * np.pi / L[0] * 0.75)
    one = _run(mesh, **kw)
    nshell = len(one.bispec.edges["k1"]) - 1
    assert nshell >= 12
    monkeypatch.setenv("NBK_BISPEC_RESIDENT", "7")
    blk = _run(mesh, **kw)
    assert blk.attrs["transforms"] > one.attrs["transforms"] == 2 * nshell
    want = bo.fft_form(_half(mesh), N, L, one.bispec.edges["k1"])
    np.testing.assert_array_equal(blk.bispec["triangles"], one.bispec["triangles"])
    B1, _ = _flat(one, want["triples"])
    B2, _ = _flat(blk, want["triples"])
    ok = want["triangles"] > 0
    assert (np.abs(B2 - B1)[ok] <= 1e-13 * want["bound"][ok]).all()
    monkeypatch.setenv("NBK_BISPEC_RESIDENT", "2")
    with pytest.raises(MemoryError, match="NBK_BISPEC_RESIDENT"):
        _run(mesh, **kw)


def test_empty_shells_and_kmax_beyond_corner(cuda):
    N, L = (16, 16, 16), (100., 100., 100.)
    mesh = _mesh(_field(N, 16), L, "f8")
    kf = 2 * np.pi / L[0]
    # dk below the fundamental: many shells hold no mode
    r = _run(mesh, dk=0.3 * kf, kmin=0.2 * kf, kmax=4.0 * kf)
    kedges = r.bispec.edges["k1"]
    want = bo.fft_form(_half(mesh), N, L, kedges)
    assert (r.power["modes"] == 0).any()
    _check(r, want, TOL["f8"], "empty shells")
    # kmax beyond the corner of k-space (sqrt(3) k_Nyquist): the outer shells are empty
    corner = np.sqrt(3) * np.pi * N[0] / L[0]
    r = _run(mesh, dk=2 * kf, kmax=1.5 * corner)
    kedges = r.bispec.edges["k1"]
    assert kedges[-1] > corner
    want = bo.fft_form(_half(mesh), N, L, kedges)
    _check(r, want, TOL["f8"], "kmax beyond the corner")
    assert (r.bispec["triangles"][-1] == 0).all() and np.isnan(r.bispec["B"][-1]).all()


def _on_ranks(comm, gid, cap):
    from test_gpu_rank_statistics import GEOMS
    N, L, _, _ = GEOMS[gid]
    if cap:
        os.environ["NBK_BISPEC_RESIDENT"] = str(cap)
    r = _run(_mesh(_field(N, 17), L, "f8", comm))
    return dict(B=r.bispec["B"], T=r.bispec["triangles"], power=r.power["power"], modes=r.power["modes"],
                transforms=r.attrs["transforms"])


@pytest.mark.parametrize("gid", ["32-P2", "32-P4", "48x36x30-P3", "44x22x26-P2"])
def test_ranks_match_one(cuda, gid):
    from test_gpu_rank_statistics import GEOMS
    from test_gpu_slab_route import _spawn
    N, L, P, _ = GEOMS[gid]
    mesh = _mesh(_field(N, 17), L, "f8")
    one = _run(mesh)
    want = bo.fft_form(_half(mesh), N, L, one.bispec.edges["k1"])
    cap = 6 if gid == "32-P2" else 0          # one geometry also takes the blocked path on every rank
    parts = _spawn(_on_ranks, P, gid, cap)
    i, j, l = want["triples"].T
    ok = want["triangles"] > 0
    for r, part in enumerate(parts):
        np.testing.assert_array_equal(part["T"], one.bispec["triangles"], err_msg="%s rank %d" % (gid, r))
        err = np.abs(part["B"][i, j, l] - one.bispec["B"][i, j, l])[ok]
        assert (err <= 1e-12 * want["bound"][ok]).all(), "%s rank %d" % (gid, r)
        np.testing.assert_array_equal(part["modes"], one.power["modes"])
        np.testing.assert_allclose(part["power"], one.power["power"], rtol=1e-12)
        if cap:
            assert part["transforms"] > one.attrs["transforms"]


def test_two_gpu_bispectrum_matches_one_gpu():
    """launches tests/mgpu_check_bispectrum.py under torchrun when the box has >= 2 GPUs"""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(ROOT, "tests", "mgpu_check_bispectrum.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    sys.stdout.write(out.stdout[-3000:])
    sys.stderr.write(out.stderr[-3000:])
    assert out.returncode == 0
