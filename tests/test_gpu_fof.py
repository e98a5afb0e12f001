"""Friends-of-friends groups (FOF, find_features) on the GPU against the CPU restatement in oracle/fof_oracle.py: the
reference's own cases (nbodykit/algorithms/tests/test_fof.py), catalogues checked label for label, edge cases, and
P = 2 and 3 processes over gloo sharing device 0 that must reproduce one rank; tests/mgpu_check_fof.py runs the same
comparison under torchrun on several GPUs."""
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

from oracle import fof_oracle as fo  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _grid(n, L, shift=0.5):
    """the particle grid of pmesh's generate_uniform_particle_grid: one particle per cell at (i + shift) L / n"""
    i = (np.arange(n) + shift) * (L / n)
    return np.stack(np.meshgrid(i, i, i, indexing="ij"), -1).reshape(-1, 3)


def _cat(pos, comm=None, **kw):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ArrayCatalog
    data = {"Position": torch.as_tensor(np.ascontiguousarray(pos)).cuda()}
    for k, v in list(kw.items()):
        if isinstance(v, np.ndarray) and len(v) == len(pos) and k != "BoxSize":
            data[k] = torch.as_tensor(np.ascontiguousarray(v)).cuda()
            del kw[k]
    return ArrayCatalog(data, comm=comm or SelfComm(), **kw)


def _lognormal(seed=42):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.cosmology import NoWiggleEHPower
    from nbodykit_b200.lab import LogNormalCatalog
    return LogNormalCatalog(Plin=NoWiggleEHPower(), nbar=3e-3, BoxSize=128., Nmesh=32, seed=seed, comm=SelfComm())


def _np(col):
    c = col.compute() if hasattr(col, "compute") else col
    return c.detach().cpu().numpy() if isinstance(c, torch.Tensor) else np.asarray(c)


# ---- the reference's cases -------------------------------------------------------------------------------------------
def test_unit_grid_every_particle_its_own_group(cuda):
    from nbodykit_b200.lab import FOF
    cat = _cat(_grid(8, 8.), BoxSize=[8., 8., 8.], Nmesh=[8, 8, 8])
    fof = FOF(cat, linking_length=0.9, nmin=0)
    assert fof.labels.dtype == np.int32
    assert fof.labels.max() == cat.csize and fof.labels.min() == 1
    # equal sizes: ordered by the smallest member, i.e. row order
    np.testing.assert_array_equal(fof.labels, np.arange(1, cat.csize + 1))
    assert fof.max_label == [cat.csize]


def test_four_shifted_grids_merge_into_groups_of_four(cuda):
    from nbodykit_b200.lab import FOF
    Q = _grid(8, 8., shift=0)
    pos = np.concatenate([Q, Q + 0.01, Q - 0.01, Q + 0.02])
    fof = FOF(_cat(pos, BoxSize=[8., 8., 8.], Nmesh=[8, 8, 8]), linking_length=0.011 * 3 ** 0.5, nmin=0, absolute=True)
    assert fof.labels.max() == 512 and fof.labels.min() == 1
    assert (np.bincount(fof.labels)[1:] == 4).all()
    np.testing.assert_array_equal(fof.labels, fo.fof_labels(pos, 0.011 * 3 ** 0.5, 0, [8.] * 3))


def test_fully_connected_grid(cuda):
    from nbodykit_b200.lab import FOF
    fof = FOF(_cat(_grid(4, 4., shift=0), BoxSize=[4., 4., 4.], Nmesh=[4, 4, 4]), linking_length=2, nmin=63, absolute=True)
    np.testing.assert_array_equal(fof.labels, 1)


def test_nonperiodic_shift_moves_features_by_the_shift(cuda):
    from nbodykit_b200.lab import FOF
    src = _lognormal()
    pos = _np(src["Position"]).astype("f8")
    vel = _np(src["Velocity"])
    dens = np.random.RandomState(3).uniform(size=len(pos))
    out = []
    for shift in (-100., 100.):
        cat = _cat(pos + shift, Velocity=vel, Density=dens)
        fof = FOF(cat, linking_length=0.2, nmin=20, periodic=False, absolute=True)
        out.append(fof.find_features(peakcolumn="Density"))
    a, b = out
    np.testing.assert_array_equal(_np(a["Length"]), _np(b["Length"]))
    for k in ("CMPosition", "PeakPosition"):
        np.testing.assert_allclose(_np(a[k])[1:] + 200., _np(b[k])[1:], rtol=1e-6)
    for k in ("CMVelocity", "PeakVelocity"):
        np.testing.assert_allclose(_np(a[k])[1:], _np(b[k])[1:], rtol=1e-6)


# ---- catalogues against the oracle -----------------------------------------------------------------------------------
def _check_against_oracle(pos, vel, box, b, nmin, periodic=True, peak=None):
    from nbodykit_b200.lab import FOF
    kw = dict(Velocity=vel)
    if peak is not None:
        kw["Density"] = peak
    if periodic:
        kw["BoxSize"] = np.asarray(box, "f8")
    fof = FOF(_cat(pos, **kw), linking_length=b, nmin=nmin, absolute=True, periodic=periodic)
    want = fo.fof_labels(pos, b, nmin, box if periodic else None)
    np.testing.assert_array_equal(fof.labels, want)
    cat = fof.find_features(peakcolumn="Density" if peak is not None else None)
    ref = fo.features(want, pos, vel, box if periodic else None, peak=peak)
    assert _np(cat["Length"])[0] == 0
    np.testing.assert_array_equal(_np(cat["Length"]), ref["Length"])
    assert _np(cat["CMPosition"]).dtype == np.float32 and _np(cat["Length"]).dtype == np.int32
    scale = float(np.max(box)) if periodic else float(np.ptp(pos))
    for k in ("CMPosition", "PeakPosition"):
        if k in ref:
            got, exp = _np(cat[k])[1:].astype("f8"), ref[k][1:]
            if periodic:
                d = np.abs(got - exp)
                d = np.minimum(d, np.asarray(box) - d)
            else:
                d = np.abs(got - exp)
            assert d.max(initial=0) <= 2e-6 * scale, k
    for k in ("CMVelocity", "PeakVelocity"):
        if k in ref:
            np.testing.assert_allclose(_np(cat[k])[1:], ref[k][1:], rtol=2e-6, atol=2e-6 * np.abs(vel).max())
    return fof, cat


def test_lognormal_catalogue(cuda):
    src = _lognormal()
    pos, vel = _np(src["Position"]), _np(src["Velocity"])
    b = 0.2 * (128. ** 3 / len(pos)) ** (1 / 3.)
    fof, _ = _check_against_oracle(pos, vel, [128.] * 3, b, 20, peak=np.random.RandomState(5).uniform(size=len(pos)))
    assert fof.labels.max() > 5


def test_lognormal_relative_linking_length(cuda):
    from nbodykit_b200.lab import FOF
    src = _lognormal()
    pos = _np(src["Position"])
    fof = FOF(src, linking_length=0.2, nmin=20)
    b = 0.2 * (128. ** 3 / src.csize) ** (1 / 3.)
    np.testing.assert_array_equal(fof.labels, fo.fof_labels(pos, b, 20, [128.] * 3))
    assert fof.attrs == dict(linking_length=0.2, nmin=20, absolute=False, periodic=True, domain_factor=1)


@pytest.mark.parametrize("dtype", ["f4", "f8"])
def test_uniform_and_clustered_noncubic_box(cuda, dtype):
    rng = np.random.RandomState(7)
    box = np.array([30., 20., 12.])
    n = 20000
    pos = rng.uniform(size=(n, 3)) * box
    # a few tight clumps
    centres = rng.uniform(size=(30, 3)) * box
    clump = (centres[rng.randint(0, 30, 6000)] + rng.normal(scale=0.3, size=(6000, 3))) % box
    pos = np.concatenate([pos, clump]).astype(dtype)
    vel = rng.normal(size=pos.shape).astype("f4")
    _check_against_oracle(pos, vel, box, 0.35, 5, peak=rng.uniform(size=len(pos)))


def test_nonperiodic_catalogue(cuda):
    rng = np.random.RandomState(8)
    pos = rng.normal(scale=4.0, size=(15000, 3)).astype("f4")
    vel = rng.normal(size=pos.shape).astype("f4")
    _check_against_oracle(pos, vel, None, 0.3, 3, periodic=False)


# ---- edge cases ------------------------------------------------------------------------------------------------------
def test_dense_blob_in_a_few_cells(cuda):
    rng = np.random.RandomState(9)
    blob = 50. + rng.uniform(-0.05, 0.05, size=(20000, 3))
    far = rng.uniform(size=(3000, 3)) * 100.
    pos = np.concatenate([blob, far])
    _check_against_oracle(pos, np.zeros_like(pos), [100.] * 3, 0.5, 10)


def test_positions_on_cell_faces_and_wrapping(cuda):
    from nbodykit_b200.lab import FOF
    L, b = 10., 0.8
    # chains along each axis across the periodic face, at L - eps / -eps, and on exact cell faces
    eps = 1e-3
    pos = np.array([[L - eps, 5, 5], [-eps, 5.4, 5], [0.3, 5, 5],               # one group across x = 0
                    [5, L - 0.2, 2], [5, 0.45, 2],                              # across y = 0
                    [2, 2, -0.1], [2, 2, L + 0.5],                              # outside [0, L): wrapped
                    [7, 7, 7]])
    ncell = int(np.ceil(L * np.sqrt(3) * (1 + 1e-9) / b))
    face = np.arange(3, 9) * (L / ncell)                       # exactly on the faces of cells 3 .. 8
    pos = np.concatenate([pos, np.stack([face, np.full(6, 8.5), np.full(6, 8.5)], 1)])
    want = fo.fof_labels(pos, b, 1, [L] * 3)
    fof = FOF(_cat(pos, BoxSize=[L] * 3), linking_length=b, nmin=1, absolute=True)
    np.testing.assert_array_equal(fof.labels, want)
    assert want[0] == want[1] == want[2] != 0 and want[3] == want[4] != 0 and want[5] == want[6] != 0


@pytest.mark.parametrize("b", [3.5, 6.0])
def test_linking_length_above_a_third_of_the_box(cuda, b):
    rng = np.random.RandomState(10)
    pos = rng.uniform(size=(300, 3)) * 10.
    pos[:, 1] *= 0.1                     # keep some structure left to find
    _check_against_oracle(pos, rng.normal(size=pos.shape), [10.] * 3, b, 2)


def test_single_particle(cuda):
    from nbodykit_b200.lab import FOF
    fof = FOF(_cat(np.array([[1., 2., 3.]]), Velocity=np.array([[1., 1., 1.]]), BoxSize=[4.] * 3), 0.5, 0, absolute=True)
    np.testing.assert_array_equal(fof.labels, [1])
    cat = fof.find_features()
    np.testing.assert_array_equal(_np(cat["Length"]), [0, 1])
    np.testing.assert_allclose(_np(cat["CMPosition"])[1], [1, 2, 3])


def test_permuted_input_same_partition(cuda):
    from nbodykit_b200.lab import FOF
    src = _lognormal(seed=3)
    pos = _np(src["Position"])
    b = 0.2 * (128. ** 3 / len(pos)) ** (1 / 3.)
    a = FOF(_cat(pos, BoxSize=[128.] * 3), b, 20, absolute=True).labels
    p = np.random.RandomState(1).permutation(len(pos))
    c = FOF(_cat(pos[p], BoxSize=[128.] * 3), b, 20, absolute=True).labels
    inv = np.empty_like(p)
    inv[p] = np.arange(len(p))
    # same sizes, and the same partition up to renaming of the labels
    np.testing.assert_array_equal(np.sort(np.bincount(a)[1:]), np.sort(np.bincount(c)[1:]))
    ca = c[inv]
    pairs = set(zip(a.tolist(), ca.tolist()))
    assert len(pairs) == len(set(a.tolist())) == len(set(ca.tolist()))


def test_two_runs_bit_identical(cuda):
    from nbodykit_b200.lab import FOF
    src = _lognormal(seed=4)
    outs = []
    for _ in range(2):
        f = FOF(src, linking_length=0.2, nmin=5)
        outs.append((f.labels, f.find_features()))
    np.testing.assert_array_equal(outs[0][0], outs[1][0])
    for k in ("CMPosition", "CMVelocity", "Length"):
        assert np.array_equal(_np(outs[0][1][k]), _np(outs[1][1][k]), equal_nan=True)


# ---- several ranks over gloo on device 0 -----------------------------------------------------------------------------
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


def _fof_ranks(comm, pos, vel, box, b, nmin, split):
    """rank r takes rows [split[r], split[r+1]) (empty ranks allowed)"""
    from nbodykit_b200.lab import ArrayCatalog, FOF
    mine = slice(split[comm.rank], split[comm.rank + 1])
    kw = dict(BoxSize=np.asarray(box, "f8")) if box is not None else {}
    cat = ArrayCatalog({"Position": torch.from_numpy(pos[mine]).cuda(), "Velocity": torch.from_numpy(vel[mine]).cuda(),
                        "InitialPosition": torch.from_numpy(pos[mine] * 0.5).cuda(),
                        "Density": torch.from_numpy(_peak(len(pos))[mine]).cuda()}, comm=comm, **kw)
    fof = FOF(cat, linking_length=b, nmin=nmin, absolute=True, periodic=box is not None)
    feat = fof.find_features(peakcolumn="Density")
    return dict(labels=fof.labels, max_label=fof.max_label, **{k: _np(feat[k]) for k in _FEATURES + ("Length",)})


_FEATURES = ("CMPosition", "CMVelocity", "InitialPosition", "PeakPosition", "PeakVelocity")


def _peak(n):
    return np.random.RandomState(17).uniform(size=n)


def _multi_case(name):
    rng = np.random.RandomState(12)
    L = 24.
    if name == "spanning":
        # a filament along x through every slab, plus background and clumps
        t = np.linspace(0, L, 400, endpoint=False)
        fil = np.stack([t, 12 + 0.05 * np.sin(t), 12 + 0.05 * np.cos(t)], 1)
        bg = rng.uniform(size=(4000, 3)) * L
        pos = np.concatenate([bg, fil]).astype("f4")
        pos = pos[np.argsort(pos[:, 0], kind="stable")]          # slab-local rows, like a generated catalogue
        return pos, [L] * 3, 0.6, 2
    if name == "wide":
        pos = (rng.uniform(size=(60, 3)) * L).astype("f4")
        return pos, [L] * 3, 9.0, 1                                # b wider than a slab (8 at P = 3) and above L / 3
    if name == "nonperiodic":
        pos = rng.normal(scale=5., size=(5000, 3)).astype("f4")
        return pos, None, 0.45, 2
    raise KeyError(name)


@pytest.mark.parametrize("P,name,empty", [(2, "spanning", False), (3, "spanning", True), (3, "wide", False),
                                          (2, "nonperiodic", False)])
def test_several_ranks_equal_one(cuda, P, name, empty):
    from nbodykit_b200.lab import FOF
    pos, box, b, nmin = _multi_case(name)
    vel = np.random.RandomState(2).normal(size=pos.shape).astype("f4")
    n = len(pos)
    split = [r * n // P for r in range(P + 1)]
    if empty:
        split = [0, 0] + [n * (r + 1) // (P - 1) for r in range(P - 1)]   # rank 0 holds nothing
    parts = _spawn(_fof_ranks, P, pos, vel, box, b, nmin, split)
    kw = dict(Velocity=vel, InitialPosition=pos * 0.5, Density=_peak(len(pos)))
    if box is not None:
        kw["BoxSize"] = np.asarray(box, "f8")
    one = FOF(_cat(pos, **kw), linking_length=b, nmin=nmin, absolute=True, periodic=box is not None)
    feat = one.find_features(peakcolumn="Density")
    np.testing.assert_array_equal(np.concatenate([p["labels"] for p in parts]), one.labels)
    np.testing.assert_array_equal(one.labels, fo.fof_labels(pos, b, nmin, box))
    assert [max(p["max_label"]) for p in parts] == [one.labels.max()] * P
    np.testing.assert_array_equal(np.concatenate([p["Length"] for p in parts]), _np(feat["Length"]))
    for k in _FEATURES:
        got = np.concatenate([p[k] for p in parts])[1:]
        np.testing.assert_allclose(got, _np(feat[k])[1:], rtol=1e-6, atol=1e-6 * (box[0] if box else 10.))
    if name == "spanning":
        assert np.bincount(one.labels)[1:].max() >= 400          # the filament is one group across all slabs


def test_two_gpu_fof_matches_one_gpu():
    """launches tests/mgpu_check_fof.py under torchrun when the box has >= 2 GPUs"""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29527", os.path.join(ROOT, "tests", "mgpu_check_fof.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    sys.stdout.write(out.stdout[-3000:])
    sys.stderr.write(out.stderr[-3000:])
    assert out.returncode == 0
