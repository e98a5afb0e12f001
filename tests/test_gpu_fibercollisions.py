"""FiberCollisions on the GPU against the restatement of oracle/fibercollisions_oracle.py with the hashed chooser: Label,
Collided and NeighborID bit for bit from `r.source['Position']`, on the reference test's catalogue, uniform fields below
and near percolation, clustered catalogues whose groups run through the warp, block and global-scratch greedy, float32
and float64 ra/dec in degrees and radians, ra across 0/360 and rows at the poles, tiny catalogues; the reference's
issue-584 rows; the golden fixtures made with the reference's code; and P = 2 and 3 processes over gloo sharing device 0,
which must reproduce one rank.  tests/mgpu_check_fibercollisions.py runs the same comparison under torchrun."""
import datetime
import glob
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import fibercollisions_oracle as fo

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RAD62 = 62 / 60. / 60.


def _run(ra, dec, comm=None, **kw):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import FiberCollisions
    return FiberCollisions(ra, dec, comm=comm or SelfComm(), **kw)


def _np(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _columns(r):
    return [_np(r.labels[c].compute()) for c in ('Label', 'Collided', 'NeighborID')]


def _check(ra, dec, seed=5, **kw):
    r = _run(ra, dec, seed=seed, **kw)
    lab, col, nb = _columns(r)
    assert lab.dtype == np.int32 and col.dtype == np.int32 and nb.dtype == np.int32
    pos = r.source['Position'].compute().cpu().numpy()
    want = fo.fiber_collisions(pos, r._collision_radius_rad, seed)
    np.testing.assert_array_equal(lab, want[0])
    np.testing.assert_array_equal(col, want[1])
    np.testing.assert_array_equal(nb, want[2])
    return r, pos


def _uniform(rng, n, ra0, ra1, dec0, dec1):
    ra = rng.uniform(ra0, ra1, n)
    dec = np.rad2deg(np.arcsin(rng.uniform(np.sin(np.deg2rad(dec0)), np.sin(np.deg2rad(dec1)), n)))
    return ra, dec


def test_reference_catalogue(cuda):
    np.random.seed(42)
    ra = 10. * np.random.random(size=10000)
    dec = 5. * np.random.random(size=10000) - 5.0
    r, pos = _check(ra, dec, seed=42)
    lab, col, nb = _columns(r)
    fo.check_invariants(pos, lab, col, nb, r._collision_radius_rad)
    s = r._stats
    assert s['groups'] == 773 and s['pairs'] == 684 and s['multiplets'] == 89 and s['largest'] == 5
    assert s['collided'] == col.sum() and 780 < col.sum() < 860
    assert r.attrs == {'collision_radius': RAD62, 'seed': 42, 'degrees': True}
    assert set(r.labels.columns) >= {'Label', 'Collided', 'NeighborID'}


@pytest.mark.parametrize("density", [1000, 4000])
def test_uniform_fields(cuda, density):
    """below and near the percolation density of the 62 arcsecond radius"""
    rng = np.random.RandomState(density)
    ra, dec = _uniform(rng, int(density * 2.5 * 2.5), 100., 102.5, 20., 22.5)
    r, _ = _check(ra, dec, seed=11)
    if density == 4000:
        assert r._stats['largest'] > 32 and r._stats['list_entries'] > 0


def _clumps(rng, sizes, sigma):
    ras, decs = [rng.uniform(200, 204, 3000)], [rng.uniform(-2, 2, 3000)]
    for k, sz in enumerate(sizes):
        c = np.array([200.3 + 0.9 * (k % 4), -1.5 + 0.9 * (k // 4)])
        ras.append(c[0] + rng.normal(scale=sigma, size=sz))
        decs.append(c[1] + rng.normal(scale=sigma, size=sz))
    return np.concatenate(ras), np.concatenate(decs)


def test_clustered_groups_beyond_shared_memory(cuda):
    """groups of 3 .. 32 members (warp), hundreds (shared-memory block) and more than nbk_fc_smem_members (global
    scratch), with many members that collide with hundreds of others"""
    from nbodykit_b200._lib import lib
    cap = int(lib().nbk_fc_smem_members())
    rng = np.random.RandomState(3)
    ra, dec = _clumps(rng, [40, 120, 700, cap + 900], 0.04)
    r, pos = _check(ra, dec, seed=7)
    lab, col, nb = _columns(r)
    sizes = np.bincount(lab)[1:]
    assert sizes.max() > cap and ((sizes > 32) & (sizes <= cap)).any()
    fo.check_invariants(pos, lab, col, nb, r._collision_radius_rad)


@pytest.mark.parametrize("dtype", ["f4", "f8"])
@pytest.mark.parametrize("degrees", [True, False])
def test_dtypes_and_radians(cuda, dtype, degrees):
    rng = np.random.RandomState(9)
    ra, dec = _uniform(rng, 20000, 10., 13., 40., 43.)
    if not degrees:
        ra, dec = np.deg2rad(ra), np.deg2rad(dec)
    _check(ra.astype(dtype), dec.astype(dtype), seed=2, degrees=degrees)


def test_wrap_in_ra_and_poles(cuda):
    rng = np.random.RandomState(10)
    ra = np.concatenate([rng.uniform(-0.5, 0.5, 6000) % 360., rng.uniform(0, 360, 50), rng.uniform(0, 360, 40),
                         rng.uniform(0, 360, 3000)])
    dec = np.concatenate([rng.uniform(-0.5, 0.5, 6000), np.full(50, 90.), np.full(40, -90.),
                          90. - rng.uniform(0, 0.7, 3000) ** 2])
    r, _ = _check(ra, dec, seed=13)
    lab, col, _ = _columns(r)
    # every row at a pole is one point: one group per pole, all but one member collided
    for sl in (slice(6000, 6050), slice(6050, 6090)):
        assert len(set(lab[sl])) == 1 and lab[sl][0] > 0


@pytest.mark.parametrize("n", [0, 1, 2])
def test_tiny_catalogues(cuda, n):
    ra, dec = np.array([10., 10.001])[:n], np.array([5., 5.])[:n]
    r, _ = _check(ra, dec, seed=1)
    lab, col, nb = _columns(r)
    assert len(lab) == n and col.sum() == (1 if n == 2 else 0)


def test_no_collisions(cuda):
    ra, dec = np.meshgrid(np.arange(0., 10., 0.1), np.arange(-5., 5., 0.1))
    r, _ = _check(ra.ravel(), dec.ravel(), seed=4)
    lab, col, nb = _columns(r)
    assert (lab == 0).all() and (col == 0).all() and (nb == -1).all()


@pytest.mark.parametrize("seed", [None, 0, 1, 2, 3])
def test_issue584(cuda, seed):
    for ra, want in (([0., 1., 2.], [0, 1, 0]), ([0., 1., 2., 10.], [0, 1, 0, 0])):
        r = _run(np.array(ra), np.zeros(len(ra)), collision_radius=1.5, seed=seed)
        _, col, nb = _columns(r)
        np.testing.assert_array_equal(col, want)
        np.testing.assert_array_equal(nb, [-1, 0] + [-1] * (len(ra) - 2))


def test_seed_none_is_recorded_and_reproduces(cuda):
    rng = np.random.RandomState(14)
    ra, dec = _uniform(rng, 8000, 50., 52., 0., 2.)
    a = _run(ra, dec, seed=None)
    assert 0 <= a.attrs['seed'] < 2 ** 32
    b = _run(ra, dec, seed=a.attrs['seed'])
    for x, y in zip(_columns(a), _columns(b)):
        np.testing.assert_array_equal(x, y)


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "fibercollisions_*.npz"))))
def test_golden_fixtures(cuda, path):
    """the reference's own output: Label everywhere, Collided and NeighborID where no random choice was made"""
    z = np.load(path)
    r = _run(z["ra"], z["dec"], collision_radius=float(z["collision_radius"]), seed=int(z["seed"]))
    lab, col, nb = _columns(r)
    np.testing.assert_array_equal(lab, z["Label"])
    f = z["forced"]
    np.testing.assert_array_equal(col[f], z["Collided"][f])
    np.testing.assert_array_equal(nb[f], z["NeighborID"][f])
    assert col.sum() == np.count_nonzero(col) and (col[lab == 0] == 0).all()


def test_golden_fixtures_exist():
    assert len(glob.glob(os.path.join(ROOT, "tests", "golden", "fibercollisions_*.npz"))) >= 4


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


def _fc_ranks(comm, ra, dec, split):
    mine = slice(split[comm.rank], split[comm.rank + 1])
    r = _run(ra[mine], dec[mine], comm=comm, seed=21)
    return _columns(r)


@pytest.mark.parametrize("P,empty", [(2, False), (3, True), (2, True)])
def test_several_ranks_equal_one(cuda, P, empty):
    rng = np.random.RandomState(15)
    ra, dec = _clumps(rng, [60, 400], 0.04)
    one = _columns(_run(ra, dec, seed=21))
    n = len(ra)
    split = list(np.linspace(0, n, P + 1).astype(int))
    if empty:
        split = [0, 0, n] if P == 2 else [0, n // 3, n // 3, n]
    res = _spawn(_fc_ranks, P, ra, dec, split)
    for k in range(3):
        np.testing.assert_array_equal(np.concatenate([r[k] for r in res]), one[k])
