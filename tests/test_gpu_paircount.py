"""Pair counts (SimulationBoxPairCount, SimulationBox2PCF) on the GPU against the CPU restatement in
oracle/paircount_oracle.py: npairs exactly equal, the double sums to rtol 1e-12.  Covers every mode, periodic or not,
auto and cross, f4 / f8 / mixed positions, weights, clustered catalogues, pairs on bin edges, positions at 0, L and
below 0, a stencil that wraps onto itself, both histogram paths, permuted input, the estimators, and P = 2 and 3
processes over gloo sharing device 0; tests/mgpu_check_paircount.py runs the same comparison under torchrun."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import paircount_oracle as po  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_COMM = []


def _comm():
    from nbodykit_b200.comm import SelfComm
    if not _COMM:
        _COMM.append(SelfComm())
    return _COMM[0]


def _cat(pos, w=None, box=None, comm=None):
    from nbodykit_b200.lab import ArrayCatalog
    data = {"Position": torch.as_tensor(np.ascontiguousarray(pos)).cuda()}
    if w is not None:
        data["Weight"] = torch.as_tensor(np.ascontiguousarray(w)).cuda()
    kw = dict(BoxSize=np.asarray(box, "f8")) if box is not None else {}
    return ArrayCatalog(data, comm=comm or _comm(), **kw)


def _np(col):
    c = col.compute() if hasattr(col, "compute") else col
    return c.detach().cpu().numpy() if isinstance(c, torch.Tensor) else np.asarray(c)


def _kw(mode, Nmu=None, pimax=None):
    return dict(Nmu=(Nmu or 6) if mode == "2d" else None, pimax=(pimax or 12.) if mode == "projected" else None)


def _compare(r, want):
    p = r.pairs
    np.testing.assert_array_equal(p["npairs"], want["npairs"])
    assert p["npairs"].dtype == np.uint64
    np.testing.assert_allclose(p["wnpairs"], want["wnpairs"], rtol=1e-12, atol=0)
    n = want["npairs"]
    sep = np.where(n > 0, want["sepsum"] / np.maximum(n, 1), 0.)
    np.testing.assert_allclose(p[p.dims[0]], sep, rtol=1e-12, atol=0)


def _run(mode, pos1, edges, box, periodic=True, pos2=None, w1=None, w2=None, los=2, **kw):
    from nbodykit_b200.lab import SimulationBoxPairCount
    first = _cat(pos1, w1, box)
    second = _cat(pos2, w2, box) if pos2 is not None else None
    r = SimulationBoxPairCount(mode, first, edges, BoxSize=box, periodic=periodic, second=second, los=los, **kw)
    want = po.count(pos1, mode, edges, box if periodic else None, pos2=pos2, w1=w1, w2=w2, los=los, **kw)
    _compare(r, want)
    return r, want


# ---- catalogues against the oracle -----------------------------------------------------------------------------------
_CASES = [  # dtype1, dtype2 (None: auto), weights, catalogue
    ("f4", None, False, "uniform"),
    ("f8", None, True, "clustered"),
    ("f4", "f4", True, "clustered"),
    ("f8", "f4", True, "clustered"),
    ("f4", "f8", False, "uniform"),
]


@pytest.mark.parametrize("mode", ["1d", "2d", "projected"])
@pytest.mark.parametrize("periodic", [True, False])
@pytest.mark.parametrize("case", range(len(_CASES)))
def test_against_oracle(cuda, mode, periodic, case):
    d1, d2, weighted, kind = _CASES[case]
    rng = np.random.RandomState(100 + case)
    L = 60.
    if kind == "uniform":
        a = rng.uniform(size=(3000, 3)) * L
    else:
        a = po.clustered(case, L, 1500, 4, 600, 0.8)          # dense blobs: cells of hundreds of rows
    b = None if d2 is None else po.clustered(case + 7, L, 1800, 2, 400, 1.5).astype(d2)
    a = a.astype(d1)
    if not periodic:
        a = a - 20.
        b = None if b is None else b - 20.
    w1 = rng.uniform(0.5, 2., len(a)) if weighted else None
    w2 = rng.uniform(0.5, 2., len(b)) if (weighted and b is not None) else None
    edges = np.linspace(0.7, 14., 8)
    r, want = _run(mode, a, edges, [L] * 3, periodic, b, w1, w2, los=[2, 0, 1][case % 3], **_kw(mode))
    assert want["npairs"].sum() > 10000
    assert r.attrs["is_cross"] == (b is not None)


def test_reference_setup(cuda):
    """the reference's tests: UniformCatalog(nbar=3e-6, BoxSize=512, seed=42), redges = linspace(10, 150, 10)"""
    from nbodykit_b200.lab import SimulationBoxPairCount, UniformCatalog
    src = UniformCatalog(nbar=3e-6, BoxSize=512., seed=42)
    pos = _np(src["Position"])
    redges = np.linspace(10, 150, 10)
    for mode, kw in (("1d", {}), ("2d", dict(Nmu=10)), ("projected", dict(pimax=50))):
        r = SimulationBoxPairCount(mode, src, redges, periodic=True, **kw)
        _compare(r, po.count(pos, mode, redges, [512.] * 3, **kw))
        assert r.pairs["npairs"].sum() > 0
        assert r.attrs["total_wnpairs"] == 0.5 * (src.csize ** 2 - src.csize)
        r = SimulationBoxPairCount(mode, src, redges, periodic=False, **kw)
        _compare(r, po.count(pos, mode, redges, None, **kw))


# ---- exact edges and boundaries --------------------------------------------------------------------------------------
def _lattice(n):
    g = np.arange(n, dtype="f8")
    return np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)


@pytest.mark.parametrize("periodic", [True, False])
def test_unit_lattice_on_bin_edges(cuda, periodic):
    """pairs exactly on r edges, at mu = 0 and mu = 1, with |dpi| on pi edges and at pimax"""
    pos = _lattice(8)
    box = [8.] * 3
    r, want = _run("1d", pos, [1., 2., 3., 4.], box, periodic)
    assert want["npairs"][0] == 512 * 26 if periodic else want["npairs"][0] > 0
    r, want = _run("2d", pos, [1., 2., 3., 4.], box, periodic, Nmu=4)
    # mu = 0 pairs (dc = 0) sit in the first mu bin, mu = 1 pairs in the last
    assert want["npairs"][0, 0] > 0 and want["npairs"][0, -1] > 0
    r, want = _run("projected", pos, [1., 2., 3.], box, periodic, pimax=3.)
    assert want["npairs"][:, 2].sum() > 0                  # |dpi| = 2 on an edge; |dpi| = 3 = pimax never counts
    _run("projected", pos.astype("f4"), [1., 2., 3.], box, periodic, pimax=3., los=0)


@pytest.mark.parametrize("dtype", ["f4", "f8"])
def test_positions_at_box_faces(cuda, dtype):
    rng = np.random.RandomState(4)
    L = 20.
    pos = rng.uniform(size=(2000, 3)) * L
    pos[:40] = 0.
    pos[40:80, 0] = L
    pos[80:120, 1] = -1e-7
    pos[120:160, 2] = L + 1e-6
    pos[160:200] = -1e-9
    pos = pos.astype(dtype)
    for mode in ("1d", "2d", "projected"):
        _run(mode, pos, [0.5, 2., 5., 9.], [L] * 3, True, **_kw(mode, pimax=8.))


def test_self_wrapping_stencil(cuda):
    """s_max just below L / 2 in a box a few cells wide: the neighbour stencil covers every cell once"""
    rng = np.random.RandomState(5)
    L = 10.
    pos = rng.uniform(size=(1500, 3)) * L
    _run("1d", pos, [0.3, 2., 4.999], [L] * 3)
    _run("2d", pos.astype("f4"), [0.3, 2., 4.999], [L] * 3, Nmu=5)
    _run("projected", pos, [0.3, 2., 3.], [L] * 3, pimax=4.999)


def test_both_histogram_paths(cuda):
    from nbodykit_b200 import _lib
    limit = int(_lib.lib().nbk_paircount_smem_bins())
    rng = np.random.RandomState(6)
    pos = rng.uniform(size=(4000, 3)) * 50.
    edges = np.linspace(1., 12., 11)
    small = limit // 10                      # 10 x small <= limit: shared-memory histogram
    big = limit // 10 + 1                    # above the limit: global atomics
    assert 10 * small <= limit < 10 * big
    for Nmu in (small, big):
        _run("2d", pos, edges, [50.] * 3, Nmu=Nmu)


def test_permuted_input_same_counts(cuda):
    from nbodykit_b200.lab import SimulationBoxPairCount
    a = po.clustered(8, 40., 2000, 3, 500, 0.6, dtype="f4")
    w = np.random.RandomState(9).uniform(size=len(a))
    p = np.random.RandomState(10).permutation(len(a))
    edges = np.linspace(0.5, 10., 6)
    r1 = SimulationBoxPairCount("2d", _cat(a, w, [40.] * 3), edges, Nmu=5)
    r2 = SimulationBoxPairCount("2d", _cat(a[p], w[p], [40.] * 3), edges, Nmu=5)
    np.testing.assert_array_equal(r1.pairs["npairs"], r2.pairs["npairs"])
    np.testing.assert_allclose(r1.pairs["wnpairs"], r2.pairs["wnpairs"], rtol=1e-12)


# ---- correlation functions -------------------------------------------------------------------------------------------
def test_natural_estimator_uniform_catalogue(cuda):
    from nbodykit_b200.algorithms.paircount import natural_estimator
    from nbodykit_b200.lab import SimulationBox2PCF, UniformCatalog
    src = UniformCatalog(nbar=2e-4, BoxSize=200., seed=7)
    pos = _np(src["Position"])
    edges = np.linspace(5, 40, 8)
    for mode, kw in (("1d", {}), ("2d", dict(Nmu=4)), ("projected", dict(pimax=20))):
        t = SimulationBox2PCF(mode, src, edges, **kw)
        want = po.count(pos, mode, edges, [200.] * 3, **kw)
        np.testing.assert_array_equal(t.D1D2["npairs"], want["npairs"])
        # the estimator applied to the oracle's counts
        fake = type("PC", (), {})()
        fake.pairs = t.D1D2.copy()
        fake.pairs["wnpairs"] = want["wnpairs"]
        fake.attrs = dict(mode=mode, N1=src.csize, N2=None, is_cross=False, BoxSize=np.array([200.] * 3),
                          total_wnpairs=0.5 * (src.csize ** 2 - src.csize))
        np.testing.assert_allclose(t.corr["corr"], natural_estimator(fake)[1]["corr"], rtol=1e-12, atol=1e-14)
        # uniform: consistent with zero within Poisson error (ordered pairs: each unordered pair twice)
        err = np.sqrt(2. / np.maximum(want["npairs"], 1))
        assert (np.abs(t.corr["corr"]) < 6 * err + 1e-3).all(), mode
        assert t.D1R2 is None and t.D2R1 is None
        if mode == "2d":
            poles = t.corr.to_poles([0, 2])
            assert poles["corr_0"].shape == (7,)
        if mode == "projected":
            np.testing.assert_allclose(t.wp["corr"], 2 * (t.corr["corr"] * 1.).sum(-1), rtol=1e-12)


def test_landy_szalay_with_randoms_and_reused_R1R2(cuda):
    from nbodykit_b200.lab import SimulationBox2PCF, SimulationBoxPairCount
    rng = np.random.RandomState(11)
    L = 60.
    d = po.clustered(12, L, 1500, 3, 300, 1.)
    r = rng.uniform(size=(4000, 3)) * L
    edges = np.linspace(1., 12., 6)
    for periodic in (True, False):
        t = SimulationBox2PCF("1d", _cat(d, box=[L] * 3), edges, randoms1=_cat(r, box=[L] * 3), periodic=periodic)
        box = [L] * 3 if periodic else None
        DD, DR, RR = (po.count(d, "1d", edges, box), po.count(d, "1d", edges, box, pos2=r), po.count(r, "1d", edges, box))
        nd, nr = len(d), len(r)
        fDD = (0.5 * (nr * nr - nr)) / (0.5 * (nd * nd - nd))
        fDR = (0.5 * (nr * nr - nr)) / (0.5 * nd * nr)
        want = (fDD * DD["wnpairs"] - 2 * fDR * DR["wnpairs"]) / RR["wnpairs"] + 1
        np.testing.assert_array_equal(t.D1D2["npairs"], DD["npairs"])
        np.testing.assert_array_equal(t.D1R2["npairs"], DR["npairs"])
        np.testing.assert_array_equal(t.R1R2["npairs"], RR["npairs"])
        np.testing.assert_allclose(t.corr["corr"], want, rtol=1e-12)
        RRpc = SimulationBoxPairCount("1d", _cat(r, box=[L] * 3), edges, periodic=periodic)
        u = SimulationBox2PCF("1d", _cat(d, box=[L] * 3), edges, randoms1=_cat(r, box=[L] * 3), R1R2=RRpc, periodic=periodic)
        np.testing.assert_array_equal(u.corr["corr"], t.corr["corr"])
        np.testing.assert_array_equal(u.R1R2["npairs"], t.R1R2["npairs"])


# ---- several ranks over gloo on device 0 -----------------------------------------------------------------------------
def _ranks(comm, mode, pos1, pos2, w1, box, periodic, edges, kw, split1, split2):
    from nbodykit_b200.lab import ArrayCatalog, SimulationBoxPairCount

    def cat(pos, w, split):
        mine = slice(split[comm.rank], split[comm.rank + 1])
        data = {"Position": torch.from_numpy(np.ascontiguousarray(pos[mine])).cuda()}
        if w is not None:
            data["Weight"] = torch.from_numpy(np.ascontiguousarray(w[mine])).cuda()
        return ArrayCatalog(data, comm=comm, BoxSize=np.asarray(box, "f8"))
    first = cat(pos1, w1, split1)
    second = cat(pos2, None, split2) if pos2 is not None else None
    r = SimulationBoxPairCount(mode, first, edges, periodic=periodic, second=second, **kw)
    return dict(npairs=r.pairs["npairs"], wnpairs=r.pairs["wnpairs"], sep=r.pairs[r.pairs.dims[0]])


_MULTI = [  # P, mode, periodic, cross, empty rank
    (2, "1d", True, False, False),
    (3, "2d", True, True, True),
    (3, "projected", False, True, False),
    (2, "1d", False, False, True),
]


@pytest.mark.parametrize("case", range(len(_MULTI)))
def test_several_ranks_equal_one(cuda, case):
    from test_gpu_fof import _spawn
    P, mode, periodic, cross, empty = _MULTI[case]
    L = 40.
    a = po.clustered(20 + case, L, 2500, 3, 400, 0.7, dtype="f4")
    a = a[np.argsort(a[:, 0], kind="stable")] if case % 2 else a        # slab-local rows, or rows anywhere
    b = po.clustered(30 + case, L, 2000, 2, 300, 1.) if cross else None
    w1 = np.random.RandomState(case).uniform(0.5, 2., len(a))
    edges = np.linspace(0.5, 9., 7)
    kw = _kw(mode, pimax=8.)

    def split(n):
        if empty:
            return [0, 0] + [n * (r + 1) // (P - 1) for r in range(P - 1)]
        return [r * n // P for r in range(P + 1)]
    parts = _spawn(_ranks, P, mode, a, b, w1, [L] * 3, periodic, edges, kw, split(len(a)), split(len(b)) if cross else None)
    one = po.count(a, mode, edges, [L] * 3 if periodic else None, pos2=b, w1=w1, **kw)
    for p in parts:
        np.testing.assert_array_equal(p["npairs"], one["npairs"])
        np.testing.assert_allclose(p["wnpairs"], one["wnpairs"], rtol=1e-12)
        np.testing.assert_array_equal(p["npairs"], parts[0]["npairs"])
    assert one["npairs"].sum() > 10000


def test_two_gpu_paircount_matches_one_gpu():
    """launches tests/mgpu_check_paircount.py under torchrun when the box has >= 2 GPUs"""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29531", os.path.join(ROOT, "tests", "mgpu_check_paircount.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    sys.stdout.write(out.stdout[-3000:])
    sys.stderr.write(out.stderr[-3000:])
    assert out.returncode == 0
