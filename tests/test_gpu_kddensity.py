"""KDDensity on the GPU against the restatement of oracle/kddensity_oracle.py: d bit for bit and the density to 1e-15
(device pow may differ from libm by an ulp), on uniform and clustered catalogues, the reference test's LogNormalCatalog,
the golden fixtures made with the reference's code, coincident rows, tiny catalogues, positions on and beyond the box
faces, voids, neighbours across periodic faces, grids of 1 and 2 cells per axis, and P = 2 and 3 processes over gloo
sharing device 0 that must reproduce one rank for any margin; tests/mgpu_check_kddensity.py runs the same comparison
under torchrun on several GPUs."""
import datetime
import glob
import os
import socket
import sys
import warnings

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import kddensity_oracle as ko

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cat(pos, L, comm=None):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ArrayCatalog
    return ArrayCatalog({"Position": torch.as_tensor(np.ascontiguousarray(pos)).cuda()}, comm=comm or SelfComm(), BoxSize=L)


def _run(pos, L, margin=1.0, comm=None):
    from nbodykit_b200.lab import KDDensity
    return KDDensity(_cat(pos, L, comm), margin=margin)


def _check(pos, L):
    r = _run(pos, L)
    d, dens = ko.density(pos, L)
    assert r.density.dtype == np.float64 and r.density.shape == (len(pos),)
    np.testing.assert_array_equal(r._distance, d)
    np.testing.assert_allclose(r.density, dens, rtol=1e-15, atol=0)
    return r


@pytest.mark.parametrize("dtype", ["f4", "f8"])
def test_uniform(cuda, dtype):
    rng = np.random.RandomState(1)
    r = _check((rng.uniform(size=(20000, 3)) * 100).astype(dtype), 100.)
    assert r._stats["candidates"] > 0 and np.isfinite(r.density).all()


def test_reference_lognormal(cuda):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.cosmology import NoWiggleEHPower
    from nbodykit_b200.lab import KDDensity, LogNormalCatalog
    src = LogNormalCatalog(Plin=NoWiggleEHPower(), nbar=3e-4, BoxSize=64., Nmesh=16, seed=42, comm=SelfComm())
    r = KDDensity(src)
    assert r.density.size == src.size
    pos = src["Position"].compute().cpu().numpy()
    d, dens = ko.density(pos, 64.)
    np.testing.assert_array_equal(r._distance, d)
    np.testing.assert_allclose(r.density, dens, rtol=1e-15, atol=0)


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "kddensity_*.npz"))))
def test_golden_fixtures(cuda, path):
    """the reference's own KDDensity output, stored with its inputs"""
    z = np.load(path)
    r = _run(z["pos"], float(z["BoxSize"]))
    np.testing.assert_allclose(r.density, z["density"], rtol=1e-15, atol=0)
    assert (np.isinf(r.density) == np.isinf(z["density"])).all()


def test_golden_fixtures_exist():
    assert len(glob.glob(os.path.join(ROOT, "tests", "golden", "kddensity_*.npz"))) >= 2


def test_coincident_rows_give_infinite_density(cuda):
    rng = np.random.RandomState(2)
    pos = np.concatenate([rng.uniform(size=(3000, 3)) * 50, np.full((8, 3), 7.25), np.full((7, 3), 30.5)])
    r = _check(pos, 50.)
    assert np.isinf(r.density[3000:3008]).all() and np.isfinite(r.density[3008:]).all()


@pytest.mark.parametrize("n", [0, 1, 5, 7, 8])
def test_tiny_catalogues(cuda, n):
    rng = np.random.RandomState(3)
    r = _check(rng.uniform(size=(n, 3)) * 10, 10.)
    assert len(r.density) == n
    if 0 < n < 8:
        assert (r.density == 0).all()


@pytest.mark.parametrize("dtype", ["f4", "f8"])
def test_positions_on_and_beyond_the_faces(cuda, dtype):
    L = 32.
    rng = np.random.RandomState(4)
    edge = np.array([[0., 0., 0.], [-1e-7, 5., 5.], [L * (1 - 1e-8), 1., 1.], [L, L, L], [-L, 2 * L, 3.5 * L],
                     [-0.3, 40., -100.], [31.9999999, 0., 31.9999999]])
    pos = np.concatenate([rng.uniform(size=(4000, 3)) * L, edge, rng.uniform(-L, 2 * L, size=(500, 3))]).astype(dtype)
    _check(pos, L)


def test_void_row_many_rings_away(cuda):
    rng = np.random.RandomState(5)
    L = 100.
    pos = rng.uniform(size=(30000, 3)) * L
    c = np.array([50., 50., 50.])
    pos = pos[np.linalg.norm(pos - c, axis=1) > 30.]
    pos = np.concatenate([pos, c[None, :]])
    r = _check(pos, L)
    assert r._distance[-1] > 0.25      # in units of the box


def test_sparse_neighbours_across_periodic_faces(cuda):
    rng = np.random.RandomState(6)
    L = 10.
    corner = rng.uniform(-0.4, 0.4, size=(40, 3)) % L
    pos = np.concatenate([corner, rng.uniform(size=(5, 3)) * L])
    _check(pos, L)


@pytest.mark.parametrize("n", [40, 60, 120])
def test_grids_of_one_and_two_cells(cuda, n):
    """4 rows per cell: 40 and 60 rows make 2 cells per axis, 120 make 3, 12 make 1"""
    from nbodykit_b200.algorithms import kdtree
    rng = np.random.RandomState(7 + n)
    pos = rng.uniform(size=(n, 3)) * 5
    r = _check(pos, 5.)
    assert r._stats["ncell"] == kdtree._ncell(n)[0] and r._stats["ncell"] <= 3
    assert _check(pos[:12], 5.)._stats["ncell"] == 1


def test_permuted_input_gives_permuted_output(cuda):
    rng = np.random.RandomState(8)
    pos = rng.uniform(size=(8000, 3)) * 20
    a = _run(pos, 20.)
    p = rng.permutation(len(pos))
    b = _run(pos[p], 20.)
    np.testing.assert_array_equal(a._distance[p], b._distance)
    np.testing.assert_array_equal(a.density[p], b.density)


def test_internal_query_against_owned_rows(cuda):
    """the external-query kernel returns the 8 smallest squared distances to the owned rows only"""
    from nbodykit_b200.algorithms import kdtree
    rng = np.random.RandomState(9)
    q = torch.from_numpy(rng.uniform(size=(3000, 3))).cuda()
    n_own = 2000
    grid = kdtree._Grid(q, n_own, kdtree._ncell(3000))
    qq = torch.from_numpy(rng.uniform(size=(300, 3))).cuda()
    cand = torch.zeros(1, dtype=torch.int64, device="cuda")
    knn = grid.query(qq, cand).cpu().numpy()
    a, b = qq.cpu().numpy(), q.cpu().numpy()[:n_own]
    dx = a[:, None, :] - b[None, :, :]
    dx = np.where(dx > 0.5, dx - 1, np.where(dx < -0.5, dx + 1, dx))
    d2 = (dx[..., 0] * dx[..., 0] + dx[..., 1] * dx[..., 1]) + dx[..., 2] * dx[..., 2]
    np.testing.assert_array_equal(knn, np.sort(d2, axis=1)[:, :8])


# ---- several ranks over gloo on device 0 -----------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


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
    mgr = mp.Manager()
    try:
        ret = mgr.dict()
        mp.spawn(_worker, args=(world, _free_port(), fn, args, ret), nprocs=world, join=True)
        return [ret[r] for r in range(world)]
    finally:
        mgr.shutdown()


def _kd_ranks(comm, pos, L, margins, split):
    mine = slice(split[comm.rank], split[comm.rank + 1])
    out = []
    for m in margins:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            r = _run(pos[mine], L, m, comm)
        out.append(dict(d=r._distance, density=r.density, phase2=int(comm.allreduce(r._stats["phase2_rows"]))))
    return out


def _multi_case(name):
    rng = np.random.RandomState(12)
    L = 40.
    if name == "clustered":
        centres = rng.uniform(size=(10, 3)) * L
        pos = np.concatenate([rng.uniform(size=(2000, 3)) * L,
                              (centres[rng.randint(0, 10, 2000)] + rng.normal(scale=1.0, size=(2000, 3))) % L,
                              np.full((9, 3), 0.0), rng.uniform(size=(3, 3)) * 0.01 + L / 3.])
        return pos.astype("f4"), L
    if name == "sparse":
        return rng.uniform(size=(60, 3)) * L, L
    raise KeyError(name)


MARGINS = [0.0, 0.01, 1.0, 50.0]


@pytest.mark.parametrize("P,name,empty", [(2, "clustered", False), (3, "clustered", True), (3, "sparse", False),
                                          (2, "sparse", True)])
def test_several_ranks_equal_one(cuda, P, name, empty):
    pos, L = _multi_case(name)
    one = _run(pos, L)
    d, _ = ko.density(pos, L)
    np.testing.assert_array_equal(one._distance, d)
    n = len(pos)
    split = list(np.linspace(0, n, P + 1).astype(int))
    if empty:
        split = [0, 0, n] if P == 2 else [0, n // 2, n // 2, n]
    res = _spawn(_kd_ranks, P, pos, L, MARGINS, split)
    for k, m in enumerate(MARGINS):
        np.testing.assert_array_equal(np.concatenate([r[k]["d"] for r in res]), one._distance, err_msg="margin %g" % m)
        np.testing.assert_array_equal(np.concatenate([r[k]["density"] for r in res]), one.density, err_msg="margin %g" % m)
    phase2 = [res[0][k]["phase2"] for k in range(len(MARGINS))]
    assert phase2[0] > 0 and phase2[1] > 0, phase2
    assert phase2[-1] == 0, phase2
