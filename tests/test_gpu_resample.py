"""Fourier-space resampling (`Field.resample`, behind MeshSource.compute(Nmesh=...) and preview(Nmesh=...)) at odd and
mixed sides, on complex-dtype meshes and on several ranks.  The P > 1 cases run P = 2 and 3 processes over gloo
(127.0.0.1) that all share device 0, with the NCCL-route transpose (NBK_FFT_TRANSPOSE=nccl), so the distributed exchange
is checked on one GPU; tests/mgpu_check_resample.py runs the same comparison under torchrun on several GPUs."""
import datetime
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L_BOX = 64.
PAIRS = [(32, 45), (45, 21), (21, 32), ((30, 33, 17), (24, 27, 35))]


def _band_limited(N):
    """a field whose frequencies (|j| <= 4 per axis) lie below the Nyquist frequency of every mesh here, on the grid N"""
    x = [np.arange(n) * (L_BOX / n) for n in N]
    X, Y, Z = np.meshgrid(*x, indexing='ij')
    q = 2 * np.pi / L_BOX
    return 1.5 + np.cos(2 * q * X) * np.sin(3 * q * Y + 0.3) + 0.25 * np.cos(q * (X - 2 * Y + 4 * Z))


def _n3(N):
    return [int(v) for v in np.ones(3, 'i8') * N]


def _freq(n):
    i = np.arange(n)
    return np.where(i < (n + 1) // 2, i, i - n)


def _rule(c, Ns, Nd):
    """NumPy restatement of the resampling rule on the compressed spectrum c [Sx][Sy][Sz/2+1]: per axis the destination
    index with label j takes the source mode with the same label when -m <= 2j < m, m = min(Ns, Nd); along z the indices
    0 .. m/2 map to themselves; every other destination mode is zero"""
    out = np.zeros((Nd[0], Nd[1], Nd[2] // 2 + 1), dtype=c.dtype)
    sel = []
    for d in range(2):
        m = min(Ns[d], Nd[d])
        j = _freq(Nd[d])
        keep = (2 * j >= -m) & (2 * j < m)
        sel.append((np.nonzero(keep)[0], j[keep] % Ns[d]))
    mzc = min(Ns[2], Nd[2]) // 2 + 1
    (dx, sx), (dy, sy) = sel
    out[np.ix_(dx, dy, np.arange(mzc))] = c[np.ix_(sx, sy, np.arange(mzc))]
    return out


@pytest.mark.parametrize("dtype", ["f8", "f4"])
@pytest.mark.parametrize("Ns,Nd", PAIRS)
def test_band_limited_field_is_reproduced(cuda, Ns, Nd, dtype):
    from nbodykit_b200.lab import ArrayMesh
    Ns, Nd = _n3(Ns), _n3(Nd)
    mesh = ArrayMesh(_band_limited(Ns).astype(dtype), BoxSize=L_BOX)
    want = _band_limited(Nd)
    got = mesh.compute(mode='real', Nmesh=Nd)
    assert got.value.shape == tuple(Nd)
    atol = 1e-12 if dtype == "f8" else 2e-5 * np.abs(want).max()
    np.testing.assert_allclose(got.numpy(), want, rtol=0, atol=atol)
    assert abs(got.cmean() - 1.5) < (1e-13 if dtype == "f8" else 1e-6)          # the mean is preserved
    c = mesh.compute(mode='complex', Nmesh=Nd)
    assert c.value.shape == (Nd[0], Nd[1], Nd[2] // 2 + 1)
    wc = np.fft.rfftn(want) / want.size
    np.testing.assert_allclose(c.numpy(), wc, rtol=0, atol=1e-12 if dtype == "f8" else 2e-5 * np.abs(wc).max())
    assert abs(c.value[0, 0, 0].item() - 1.5) < (1e-13 if dtype == "f8" else 1e-6)


@pytest.mark.parametrize("dtype", ["f8", "f4"])
@pytest.mark.parametrize("Ns,Nd", PAIRS + [(32, 48), (48, 32), (33, 32), (32, 33), ((16, 20, 10), (18, 15, 11))])
def test_every_destination_mode_follows_the_rule(cuda, Ns, Nd, dtype):
    """a random field, Nyquist planes included: each destination mode is an exact copy of its source mode, or zero"""
    from nbodykit_b200.lab import ArrayMesh
    Ns, Nd = _n3(Ns), _n3(Nd)
    mesh = ArrayMesh(np.random.RandomState(3).standard_normal(Ns).astype(dtype), BoxSize=L_BOX)
    src = mesh.compute(mode='complex').numpy()
    got = mesh.compute(mode='complex', Nmesh=Nd).numpy()
    assert np.array_equal(got, _rule(src, Ns, Nd))


@pytest.mark.parametrize("Ns,Nd,band", [(45, 33, False), ((21, 45, 33), (33, 27, 45), False), (32, 48, True),
                                        ((30, 33, 17), (24, 27, 35), True)])
def test_complex_dtype_mesh(cuda, Ns, Nd, band):
    """a 'c16' mesh keeps all N^3 modes: compute(mode='complex', Nmesh=M) equals fftn of the resampled real field over
    every mode.  Random fields where the smaller side is odd on every axis (the label set is symmetric, so the resampled
    spectrum is Hermitian), band-limited ones otherwise"""
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import FieldMesh
    from nbodykit_b200.pmesh.pm import ParticleMesh, RealField
    Ns, Nd = _n3(Ns), _n3(Nd)
    a = _band_limited(Ns) if band else np.random.RandomState(5).standard_normal(Ns)
    f = RealField(ParticleMesh(BoxSize=L_BOX, Nmesh=Ns, dtype='c16', comm=SelfComm()))
    f[...] = a
    mesh = FieldMesh(f)
    real = mesh.compute(mode='real', Nmesh=Nd)
    c = mesh.compute(mode='complex', Nmesh=Nd)
    assert c.value.shape == tuple(Nd) and real.value.shape == tuple(Nd)
    want = np.fft.fftn(real.numpy()) / np.prod(Nd)
    np.testing.assert_allclose(c.numpy(), want, rtol=0, atol=1e-13 * max(1.0, np.abs(want).max()))
    # and the same numbers as the compressed mesh
    ref = RealField(ParticleMesh(BoxSize=L_BOX, Nmesh=Ns, dtype='f8', comm=SelfComm()))
    ref[...] = a
    np.testing.assert_allclose(real.numpy(), FieldMesh(ref).compute(mode='real', Nmesh=Nd).numpy(), rtol=0,
                               atol=1e-13 * np.abs(a).max())


@pytest.mark.parametrize("Ns,M,axes", [(32, 45, (0, 1)), (45, 21, (2,)), ((30, 33, 17), (24, 27, 35), (1, 0)),
                                       (32, 16, None)])
def test_preview_at_another_resolution(cuda, Ns, M, axes):
    from nbodykit_b200.lab import ArrayMesh
    mesh = ArrayMesh(np.random.RandomState(9).standard_normal(_n3(Ns)), BoxSize=L_BOX)
    got = mesh.preview(Nmesh=M, axes=axes)
    want = mesh.compute(mode='real', Nmesh=M).preview(axes=axes)
    np.testing.assert_array_equal(got, want)


def test_linear_mesh_preview_of_the_mesh_guide(cuda):
    """the plotting example of the reference's mesh guide (docs/source/mesh/common-operations.ipynb)"""
    from nbodykit_b200.cosmology import NoWiggleEHPower
    from nbodykit_b200.lab import LinearMesh
    mesh = LinearMesh(NoWiggleEHPower(), BoxSize=1380., Nmesh=128, seed=42)
    img = mesh.preview(Nmesh=64, axes=(0, 1))
    assert img.shape == (64, 64) and np.isfinite(img).all()
    np.testing.assert_array_equal(img, mesh.compute(mode='real', Nmesh=64).preview(axes=(0, 1)))


# ---- several ranks on device 0 ------------------------------------------------------------------------------------

def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, fn, args, ret):
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
    """runs fn(comm, *args) on `world` processes sharing device 0 and returns their results; every process is joined
    before this returns"""
    mgr = mp.Manager()
    try:
        ret = mgr.dict()
        mp.spawn(_worker, args=(world, _free_port(), fn, args, ret), nprocs=world, join=True)
        return [ret[r] for r in range(world)]
    finally:
        mgr.shutdown()


def _gathered(field):
    """this rank's part of a field as numpy: real x slabs, or complex transposed y slabs in [Nx][y_n][Nzc] order"""
    a = field.numpy()
    from nbodykit_b200.pmesh.pm import ComplexField
    return a.transpose(1, 0, 2) if isinstance(field, ComplexField) and field.pm.transposed else a


def _compute_ranks(comm, a, M, dtype):
    from nbodykit_b200.lab import ArrayMesh
    mesh = ArrayMesh(a.astype(dtype), BoxSize=L_BOX, comm=comm)
    out = {}
    for mode in ("real", "complex"):
        out[mode] = _gathered(mesh.compute(mode=mode, Nmesh=M))
    out["preview"] = mesh.preview(Nmesh=M, axes=(0, 2))
    out["preview_all"] = mesh.preview(Nmesh=M)
    return out


@pytest.mark.parametrize("P,Ns,M", [(3, 48, 36), (3, 45, 33), (2, 32, 48)])
def test_resample_on_several_ranks_equals_one_gpu(cuda, P, Ns, M):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ArrayMesh
    a = np.random.RandomState(11).standard_normal((Ns, Ns, Ns))
    parts = _spawn(_compute_ranks, P, a, M, "f8")
    mesh = ArrayMesh(a, BoxSize=L_BOX, comm=SelfComm())
    for mode, axis in (("real", 0), ("complex", 1)):
        got = np.concatenate([p[mode] for p in parts], axis=axis)
        want = mesh.compute(mode=mode, Nmesh=M).numpy()
        assert got.shape == want.shape
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-12 * np.abs(want).max())
    for key, axes in (("preview", (0, 2)), ("preview_all", None)):
        want = mesh.preview(Nmesh=M, axes=axes)
        for p in parts:
            np.testing.assert_allclose(p[key], want, rtol=0, atol=1e-12 * np.abs(want).max())


def _fftpower_ranks(comm, pos, w):
    from nbodykit_b200.lab import ArrayCatalog, FFTPower
    mine = slice(comm.rank * len(pos) // comm.size, (comm.rank + 1) * len(pos) // comm.size)
    cat = ArrayCatalog({"Position": torch.from_numpy(pos[mine]).cuda(), "Weight": torch.from_numpy(w[mine]).cuda()},
                       comm=comm, BoxSize=L_BOX)
    r = FFTPower(cat.to_mesh(Nmesh=32, resampler="cic", compensated=True, dtype="f8"), mode="2d", Nmu=4, poles=[0, 2])
    return {k: np.asarray(r.power[k]) for k in ("k", "modes", "power")}


def test_harness_fftpower_two_ranks_equals_one(cuda):
    """the harness itself: FFTPower at 32^3 on two ranks of device 0 equals one rank"""
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ArrayCatalog, FFTPower
    rng = np.random.RandomState(21)
    pos = (rng.uniform(0, 1, size=(50000, 3)) * L_BOX).astype("f4")
    w = rng.uniform(0.5, 1.5, size=len(pos))
    parts = _spawn(_fftpower_ranks, 2, pos, w)
    cat = ArrayCatalog({"Position": torch.from_numpy(pos).cuda(), "Weight": torch.from_numpy(w).cuda()},
                       comm=SelfComm(), BoxSize=L_BOX)
    r = FFTPower(cat.to_mesh(Nmesh=32, resampler="cic", compensated=True, dtype="f8"), mode="2d", Nmu=4, poles=[0, 2])
    for p in parts:
        assert np.array_equal(p["modes"], r.power["modes"])
        np.testing.assert_allclose(np.nan_to_num(p["k"]), np.nan_to_num(r.power["k"]), rtol=1e-12)
        np.testing.assert_allclose(np.nan_to_num(p["power"]), np.nan_to_num(r.power["power"]), rtol=1e-10,
                                   atol=1e-10 * np.nanmax(np.abs(r.power["power"])))


def test_two_gpu_resample_matches_one_gpu():
    """launches tests/mgpu_check_resample.py under torchrun when the box has >= 2 GPUs"""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29523", os.path.join(ROOT, "tests", "mgpu_check_resample.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    sys.stdout.write(out.stdout[-3000:])
    sys.stderr.write(out.stderr[-3000:])
    assert out.returncode == 0
