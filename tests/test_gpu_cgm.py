"""CylindricalGroups and CatalogSource.sort on the GPU against the float64 restatement in oracle/cgm_oracle.py: the
reference's own cases (nbodykit/algorithms/tests/test_cgm.py), the golden fixtures made with the reference's code,
lines of sight, priorities, edges of the cylinder and of the box, long dependency chains, and P = 2 and 3 processes
over gloo sharing device 0 that must reproduce one rank; tests/mgpu_check_cgm.py runs the same comparison under torchrun
on several GPUs."""
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

from oracle import cgm_oracle as co

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COLS = ("cgm_type", "cgm_haloid", "num_cgm_sats")


def _cat(pos, keys, comm=None, box=None):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ArrayCatalog
    data = {"Position": torch.as_tensor(np.ascontiguousarray(pos)).cuda()}
    for k, v in keys.items():
        data[k] = torch.as_tensor(np.ascontiguousarray(v)).cuda()
    kw = {} if box is None else dict(BoxSize=np.ones(3) * np.asarray(box, "f8"))
    return ArrayCatalog(data, comm=comm or SelfComm(), **kw)


def _run(pos, keys, rankby, rperp, rpar, los=None, periodic=False, box=None, comm=None):
    from nbodykit_b200.lab import CylindricalGroups
    cat = _cat(pos, keys, comm, box if periodic else None)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        r = CylindricalGroups(cat, rankby, rperp, rpar, flat_sky_los=los, periodic=periodic,
                              BoxSize=None if periodic else box)
    return {c: np.asarray(r.groups[c].compute()) for c in COLS}, r


def _check(pos, keys, rankby, rperp, rpar, los=None, periodic=False, box=None):
    got, r = _run(pos, keys, rankby, rperp, rpar, los, periodic, box)
    ks = [keys[k] for k in ([rankby] if isinstance(rankby, str) else (rankby or []))]
    t, h, s, _ = co.cgm(pos, ks, rperp, rpar, los=los, periodic=periodic, BoxSize=box)
    assert got["cgm_type"].dtype == np.uint32 and got["cgm_haloid"].dtype == np.int64
    np.testing.assert_array_equal(got["cgm_type"], t)
    np.testing.assert_array_equal(got["cgm_haloid"], h)
    np.testing.assert_array_equal(got["num_cgm_sats"], s)
    return got, r


def _reference_case(seed=42):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import UniformCatalog
    src = UniformCatalog(3e-4, BoxSize=256, seed=seed, comm=SelfComm())
    logmass = np.asarray(src.rng.uniform(12, 15))
    gal = np.empty(len(src))
    gal[logmass < 14.5] = 0
    gal[logmass > 14.5] = 1
    pos = np.asarray(src["Position"].compute())
    return pos, {"halo_mvir": 10 ** logmass, "gal_type": gal}


# ---- the reference's cases -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("periodic", [True, False])
def test_reference_cases(cuda, periodic):
    pos, keys = _reference_case()
    got, r = _check(pos, keys, ["halo_mvir", "gal_type"], 10., 10., los=[0, 0, 1], periodic=periodic, box=256.)
    assert r.attrs["rankby"] == ["halo_mvir", "gal_type"] and list(r.attrs["BoxSize"]) == [256.] * 3
    assert (got["cgm_type"] == 1).sum() > 0


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "cgm_*.npz"))))
def test_golden_fixtures(cuda, path):
    """the reference's own cgm() (or direct_cgm) output, stored with its inputs"""
    z = np.load(path)
    los = z["los"] if z["los"].size == 3 else None
    periodic = bool(z["periodic"])
    got, _ = _run(z["pos"], {"mass": z["mass"], "gal_type": z["gal_type"]}, ["mass", "gal_type"], float(z["rperp"]),
                  float(z["rpar"]), los, periodic, float(z["box"]))
    for c in COLS:
        np.testing.assert_array_equal(got[c], z[c])


def test_golden_fixtures_exist():
    assert len(glob.glob(os.path.join(ROOT, "tests", "golden", "cgm_*.npz"))) >= 2


# ---- lines of sight --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("los", [[1, 0, 0], [0, 1, 0], [0, 0, 1], [0.48, 0.6, 0.64]])
@pytest.mark.parametrize("dtype", ["f4", "f8"])
def test_flat_sky_lines_of_sight(cuda, los, dtype):
    rng = np.random.RandomState(3)
    pos = (rng.uniform(size=(6000, 3)) * 100).astype(dtype)
    m = rng.uniform(size=6000)
    _check(pos, {"m": m}, "m", 2.0, 6.0, los=los, periodic=True, box=100.)
    _check(pos, {"m": m}, "m", 2.0, 6.0, los=los, periodic=False, box=100.)


@pytest.mark.parametrize("dtype", ["f4", "f8"])
def test_observer_at_origin_survey_shell(cuda, dtype):
    rng = np.random.RandomState(4)
    u = rng.normal(size=(8000, 3))
    u /= np.linalg.norm(u, axis=1)[:, None]
    r = rng.uniform(400, 450, size=8000)
    pos = (u * r[:, None]).astype(dtype)
    _check(pos, {"m": rng.uniform(size=8000)}, "m", 4.0, 12.0)


def test_periodic_observer_at_origin_warns(cuda):
    from nbodykit_b200.lab import CylindricalGroups
    rng = np.random.RandomState(5)
    pos = rng.uniform(size=(3000, 3)) * 50
    m = rng.uniform(size=3000)
    with pytest.warns(UserWarning):
        CylindricalGroups(_cat(pos, {"m": m}, box=50.), "m", 3., 3., periodic=True)
    _check(pos, {"m": m}, "m", 3., 3., periodic=True, box=50.)


# ---- priorities ------------------------------------------------------------------------------------------------------
def test_rankby_none_is_row_order(cuda):
    rng = np.random.RandomState(6)
    pos = rng.uniform(size=(4000, 3)) * 40
    _check(pos, {}, None, 2., 2., los=[0, 0, 1], periodic=True, box=40.)


def test_two_keys_with_ties_all_equal_and_negative(cuda):
    rng = np.random.RandomState(7)
    n = 5000
    pos = rng.uniform(size=(n, 3)) * 40
    keys = {"a": rng.randint(0, 4, size=n).astype("i4"), "b": rng.normal(size=n), "c": np.full(n, 3.0),
            "neg": -rng.uniform(1, 2, size=n), "z": np.where(rng.uniform(size=n) < 0.5, -0.0, 0.0)}
    _check(pos, keys, ["a", "b"], 2., 3., los=[0, 0, 1], periodic=True, box=40.)
    _check(pos, keys, "c", 2., 3., los=[0, 0, 1], periodic=True, box=40.)
    _check(pos, keys, "neg", 2., 3., los=[0, 0, 1], periodic=True, box=40.)
    _check(pos, keys, ["z", "a"], 2., 3., los=[0, 0, 1], periodic=True, box=40.)


def test_permuted_input_gives_permuted_output(cuda):
    rng = np.random.RandomState(8)
    n = 5000
    pos = rng.uniform(size=(n, 3)) * 40
    m = rng.uniform(size=n)
    a, _ = _run(pos, {"m": m}, "m", 2., 3., [0, 0, 1], True, 40.)
    p = rng.permutation(n)
    b, _ = _run(pos[p], {"m": m[p]}, "m", 2., 3., [0, 0, 1], True, 40.)
    for c in COLS:
        np.testing.assert_array_equal(a[c][p], b[c])


def test_nan_key_raises(cuda):
    from nbodykit_b200.lab import CylindricalGroups
    m = np.ones(10)
    m[3] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        CylindricalGroups(_cat(np.zeros((10, 3)), {"m": m}), "m", 1., 1.)


# ---- edges -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rperp,rpar", [(0., 1.), (1., 0.)])
def test_zero_radius_links_coincident_rows(cuda, rperp, rpar):
    rng = np.random.RandomState(9)
    base = rng.uniform(size=(300, 3)) * 20
    pos = np.concatenate([base, base[:100], base[:50]])
    m = rng.uniform(size=len(pos))
    got, _ = _check(pos, {"m": m}, "m", rperp, rpar, los=[0, 0, 1])
    assert (got["cgm_type"] == 1).sum() >= 100


def test_dyadic_edge_is_linked(cuda):
    """pairs exactly at rperp and at rpar (dyadic, so every operation is exact) are linked: the test is <="""
    pos = np.array([[0., 0., 0.], [0.5, 0., 0.], [10., 0., 0.], [10., 0., 0.25], [20., 0., 0.], [20.5, 0., 0.25]])
    m = np.array([6., 5., 4., 3., 2., 1.])
    got, _ = _check(pos, {"m": m}, "m", 0.5, 0.25, los=[0, 0, 1])
    np.testing.assert_array_equal(got["cgm_type"], [0, 1, 0, 1, 0, 1])
    np.testing.assert_array_equal(got["num_cgm_sats"], [1, 0, 1, 0, 1, 0])


def test_pair_symmetric_about_origin_is_not_linked(cuda):
    pos = np.array([[1., 0., 0.], [-1., 0., 0.], [0., 50., 0.5], [0., -50., -0.5]])
    got, _ = _check(pos, {"m": np.arange(4.)}, "m", 10., 10.)
    np.testing.assert_array_equal(got["cgm_type"], [0, 0, 0, 0])


def test_links_across_periodic_faces(cuda):
    rng = np.random.RandomState(10)
    L = 30.
    pos = np.concatenate([rng.uniform(size=(500, 3)) * L, rng.uniform(-0.5, 0.5, size=(400, 3)) % L,
                          np.array([[-1e-9, 15., 15.], [29.5, 15., 15.]])])
    m = rng.uniform(size=len(pos))
    got, _ = _check(pos, {"m": m}, "m", 1.0, 1.5, los=[0.6, 0, 0.8], periodic=True, box=L)
    assert (got["num_cgm_sats"] > 5).any()


def test_dense_clump(cuda):
    rng = np.random.RandomState(11)
    pos = np.concatenate([rng.normal(scale=0.05, size=(4000, 3)) + 10, rng.uniform(size=(2000, 3)) * 20])
    m = rng.uniform(size=len(pos))
    got, _ = _check(pos, {"m": m}, "m", 0.5, 0.5, los=[0, 0, 1])
    assert got["num_cgm_sats"].max() > 3000


def test_chain_needs_several_rounds(cuda):
    """a line whose priority rises along it: every row depends on the decision of the one after it"""
    n = 10000
    pos = np.zeros((n, 3))
    pos[:, 0] = np.arange(n) * 1.0
    got, r = _check(pos, {"m": np.arange(n, dtype="f8")}, "m", 1.5, 1.5, los=[0, 0, 1])
    assert r.rounds > 1
    # alternate central / satellite from the top of the line down
    np.testing.assert_array_equal(got["cgm_type"][::-1], np.arange(n) % 2)


@pytest.mark.parametrize("n", [0, 1])
def test_empty_and_single_row(cuda, n):
    got, r = _check(np.zeros((n, 3)) + 1, {"m": np.ones(n)}, "m", 1., 1., los=[0, 0, 1])
    assert len(got["cgm_type"]) == n
    if n:
        assert got["cgm_type"][0] == 0 and got["cgm_haloid"][0] == 0


# ---- CatalogSource.sort ----------------------------------------------------------------------------------------------
def _sort_expect(cols, keys, reverse):
    n = len(cols[keys[0]])
    return np.argsort(co.priority([cols[k] for k in keys], n, reverse=reverse), kind="stable")


def _sort_case(n=3000, seed=13):
    rng = np.random.RandomState(seed)
    return {"a": rng.randint(0, 5, size=n).astype("i8"), "b": rng.normal(size=n).astype("f4"),
            "Position": rng.uniform(size=(n, 3)), "row": np.arange(n)}


@pytest.mark.parametrize("reverse", [False, True])
def test_sort_one_rank(cuda, reverse):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ArrayCatalog
    cols = _sort_case()
    cat = ArrayCatalog(cols, comm=SelfComm(), BoxSize=1.0)
    out = cat.sort(["a", "b"], reverse=reverse)
    order = _sort_expect(cols, ["a", "b"], reverse)
    for k in cols:
        np.testing.assert_array_equal(np.asarray(out[k].compute()), cols[k][order])
    assert out.attrs["BoxSize"] == 1.0 and "Weight" in out
    sub = cat.sort("b", usecols=["row"])
    assert "a" not in sub.columns and "row" in sub.columns
    np.testing.assert_array_equal(np.asarray(sub["row"].compute()), _sort_expect(cols, ["b"], False))


def test_sort_errors(cuda):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ArrayCatalog
    cols = _sort_case(10)
    cols["nan"] = np.ones(10)
    cols["nan"][2] = np.nan
    cat = ArrayCatalog(cols, comm=SelfComm())
    with pytest.raises(ValueError, match="NaN"):
        cat.sort("nan")


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


def _cgm_ranks(comm, pos, keys, rankby, rperp, rpar, los, periodic, box, split):
    mine = slice(split[comm.rank], split[comm.rank + 1])
    got, r = _run(pos[mine], {k: v[mine] for k, v in keys.items()}, rankby, rperp, rpar, los, periodic, box, comm)
    return dict(got, rounds=r.rounds)


def _sort_ranks(comm, cols, keys, reverse, split):
    from nbodykit_b200.lab import ArrayCatalog
    mine = slice(split[comm.rank], split[comm.rank + 1])
    cat = ArrayCatalog({k: v[mine] for k, v in cols.items()}, comm=comm)
    out = cat.sort(keys, reverse=reverse, usecols=["row", "Position"])
    return {k: np.asarray(out[k].compute()) for k in ("row", "Position")}


def _multi_case(name):
    rng = np.random.RandomState(12)
    L = 24.
    n = 4000
    if name == "spanning":
        # a dense filament along x through every slab, plus background
        t = rng.uniform(0, L, size=600)
        fil = np.stack([t, 12 + 0.05 * np.sin(t), 12 + 0.05 * np.cos(t)], 1)
        pos = np.concatenate([rng.uniform(size=(n, 3)) * L, fil])
        return pos, {"m": rng.uniform(size=len(pos))}, "m", 0.7, 1.2, [1, 0, 0], True, L
    if name == "wide":
        pos = rng.uniform(size=(300, 3)) * L
        return pos, {"m": rng.randint(0, 3, size=300).astype("i4")}, "m", 6.0, 9.0, [0, 0, 1], True, L
    if name == "survey":
        pos = rng.normal(scale=6., size=(n, 3)) + 30
        return pos, {"m": rng.uniform(size=n)}, "m", 0.8, 2.0, None, False, None
    if name == "chain":
        pos = np.zeros((2000, 3))
        pos[:, 0] = np.arange(2000) * 0.01
        return pos, {}, None, 0.015, 0.015, [0, 0, 1], False, None
    raise KeyError(name)


@pytest.mark.parametrize("P,name,empty", [(2, "spanning", False), (3, "spanning", True), (3, "wide", False),
                                          (2, "survey", False), (3, "chain", True)])
def test_several_ranks_equal_one(cuda, P, name, empty):
    pos, keys, rankby, rperp, rpar, los, periodic, box = _multi_case(name)
    one, _ = _run(pos, keys, rankby, rperp, rpar, los, periodic, box)
    ks = [keys[k] for k in ([rankby] if isinstance(rankby, str) else (rankby or []))]
    t, h, s, _ = co.cgm(pos, ks, rperp, rpar, los=los, periodic=periodic, BoxSize=box)
    np.testing.assert_array_equal(one["cgm_type"], t)
    np.testing.assert_array_equal(one["cgm_haloid"], h)
    np.testing.assert_array_equal(one["num_cgm_sats"], s)
    n = len(pos)
    split = [0, n // 3, n // 3, n] if empty else list(np.linspace(0, n, P + 1).astype(int))
    if empty and P == 3:
        split = [0, 0, n // 2, n]
    res = _spawn(_cgm_ranks, P, pos, keys, rankby, rperp, rpar, los, periodic, box, split)
    for c in COLS:
        np.testing.assert_array_equal(np.concatenate([r[c] for r in res]), one[c])


@pytest.mark.parametrize("P", [2, 3])
@pytest.mark.parametrize("reverse", [False, True])
def test_sort_several_ranks(cuda, P, reverse):
    cols = _sort_case(2000)
    n = 2000
    split = [0, 700, 700, n] if P == 3 else [0, 1200, n]
    res = _spawn(_sort_ranks, P, cols, ["a", "b"], reverse, split)
    order = _sort_expect(cols, ["a", "b"], reverse)
    for r in range(P):
        assert len(res[r]["row"]) == split[r + 1] - split[r]
    np.testing.assert_array_equal(np.concatenate([r["row"] for r in res]), order)
    np.testing.assert_array_equal(np.concatenate([r["Position"] for r in res]), cols["Position"][order])
