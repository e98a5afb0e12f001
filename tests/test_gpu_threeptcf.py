"""The three-point function (SimulationBox3PCF) on the GPU: the reference's golden C++ result, and the CPU restatement
in oracle/threeptcf_oracle.py with npairs exactly equal and |zeta - oracle| <= 1e-9 B (B: the oracle's bound on
|zeta|).  Covers f4 / f8 positions, periodic or not, a non-cubic periodic box, uniform and clustered catalogues (cells
of hundreds of rows), signed and unit weights, e_0 = 0 and e_0 > 0, lattice separations on the bin edges, duplicate
positions, positions at 0, L and below 0, odd / even / single poles, l and the bin count at their caps, empty and
one-object catalogues, permuted input, save / load, and P = 2 and 3 processes over gloo sharing device 0 against one
(npairs identical, zeta within 1e-12 B); tests/mgpu_check_threeptcf.py runs the comparison under torchrun."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import threeptcf_oracle as to  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_COMM = []
_GOLDEN = {}


def _comm():
    from nbodykit_b200.comm import SelfComm
    if not _COMM:
        _COMM.append(SelfComm())
    return _COMM[0]


def _cat(pos, w=None, box=None, comm=None, wname="Weight"):
    from nbodykit_b200.lab import ArrayCatalog
    data = {"Position": torch.as_tensor(np.ascontiguousarray(pos)).cuda()}
    if w is not None:
        data[wname] = torch.as_tensor(np.ascontiguousarray(w)).cuda()
    kw = dict(BoxSize=np.asarray(box, "f8")) if box is not None else {}
    return ArrayCatalog(data, comm=comm or _comm(), **kw)


def _zeta(r, poles):
    return np.stack([r.poles["corr_%d" % ell] for ell in poles])


def _within(z, want, tol):
    err = np.abs(z - want["zeta"])
    assert (err <= tol * want["bound"]).all(), float(np.max(err / np.maximum(want["bound"], 1e-300)))


def _run(pos, edges, poles, box, periodic=True, w=None):
    from nbodykit_b200.lab import SimulationBox3PCF
    r = SimulationBox3PCF(_cat(pos, w, box), poles, edges, BoxSize=box, periodic=periodic)
    want = to.compute(pos, edges, poles, box=box if periodic else None, w=w)
    np.testing.assert_array_equal(r.npairs, want["npairs"])
    assert r.npairs.dtype == np.uint64
    z = _zeta(r, poles)
    _within(z, want, 1e-9)
    np.testing.assert_array_equal(z, np.swapaxes(z, 1, 2))
    assert r.candidates >= int(want["npairs"].sum())
    return r, want


# ---- the reference's golden data ------------------------------------------------------------------------------------
def _golden():
    if not _GOLDEN:
        pos, w, truth = to.golden()
        _GOLDEN.update(pos=pos, w=w, truth=truth)
    return _GOLDEN


def test_golden_cpp_result(cuda):
    """1000 weighted points in L = 400, 8 bins over [0, 200] (r_max = L / 2: 3 cells per axis, a stencil that wraps
    onto itself), l = 0 .. 10, against Daniel Eisenstein's C++ result to its 7 printed digits, and against the oracle"""
    from nbodykit_b200.lab import SimulationBox3PCF
    g = _golden()
    cat = _cat(g["pos"], g["w"], [400.] * 3, wname="w")
    edges = np.linspace(0, 200., 9)
    ells = list(range(11))
    r = SimulationBox3PCF(cat, ells, edges, BoxSize=400., weight="w")
    for i, ell in enumerate(ells):
        np.testing.assert_allclose(r.poles["corr_%d" % ell] * (4 * np.pi) ** 2 / (2 * ell + 1), g["truth"][..., i],
                                   rtol=1e-6, err_msg="l = %d" % ell)
    want = to.compute(g["pos"], edges, ells, box=[400.] * 3, w=g["w"])
    np.testing.assert_array_equal(r.npairs, want["npairs"])
    _within(_zeta(r, ells), want, 1e-9)
    # the reference test's poles, in its order
    r2 = SimulationBox3PCF(cat, [1, 0], edges, BoxSize=400., weight="w")
    assert r2.poles.variables == ["corr_1", "corr_0"]
    for ell in (1, 0):
        np.testing.assert_allclose(r2.poles["corr_%d" % ell] * (4 * np.pi) ** 2 / (2 * ell + 1), g["truth"][..., ell],
                                   rtol=1e-6)


def test_golden_pedantic_subset(cuda):
    """the reference's pedantic case: cat[::20], poles [0, 2, 4, 8]; run() and run(pedantic=True) agree"""
    from nbodykit_b200.lab import SimulationBox3PCF
    g = _golden()
    pos, w = g["pos"][::20], g["w"][::20]
    edges = np.linspace(0, 200., 9)
    poles = [0, 2, 4, 8]
    r = SimulationBox3PCF(_cat(pos, w, [400.] * 3, wname="w"), poles, edges, BoxSize=400., weight="w")
    a = _zeta(r, poles)
    b = r.run(pedantic=True)
    b = np.stack([b["corr_%d" % ell] for ell in poles])
    want = to.compute(pos, edges, poles, box=[400.] * 3, w=w)
    _within(a, want, 1e-9)
    err = np.abs(a - b)
    assert (err <= 1e-12 * want["bound"]).all()


# ---- catalogues against the oracle -----------------------------------------------------------------------------------
_CASES = [  # dtype, periodic, box, weights, catalogue, edges, poles
    ("f4", True, [30.] * 3, "unit", "uniform", np.linspace(0., 6., 5), list(range(11))),
    ("f8", True, [60.] * 3, "signed", "clustered", np.linspace(0.7, 5., 6), [0, 2, 4]),
    ("f8", False, [60.] * 3, None, "clustered", np.linspace(0., 4., 4), [1, 3]),
    ("f4", True, [30., 24., 36.], "signed", "uniform", np.linspace(0.5, 6., 4), [10]),
    ("f8", True, [30.] * 3, "signed", "uniform", np.linspace(0., 6., 33), [0, 1]),
    ("f8", False, [30.] * 3, "unit", "uniform", np.linspace(0., 5., 33), list(range(11))),
]


@pytest.mark.parametrize("case", range(len(_CASES)))
def test_against_oracle(cuda, case):
    dt, periodic, box, wkind, kind, edges, poles = _CASES[case]
    rng = np.random.RandomState(200 + case)
    L = np.asarray(box)
    if kind == "uniform":
        pos = rng.uniform(size=(3000, 3)) * L
    else:
        pos = to.clustered(case, L[0], 1200, 2, 400, 0.5)        # dense blobs: cells of hundreds of rows, split chunks
    if not periodic:
        pos = pos - 20.
    pos = pos.astype(dt)
    w = None if wkind is None else (np.ones(len(pos)) if wkind == "unit" else rng.uniform(-1., 2., len(pos)))
    r, want = _run(pos, edges, poles, box, periodic, w)
    assert want["npairs"].sum() > 20000
    if kind == "clustered":
        from nbodykit_b200 import _lib
        assert want["npairs"].sum() > 10 * int(_lib.lib().nbk_threeptcf_chunk_rows()) ** 2


def _lattice(n):
    g = np.arange(n, dtype="f8")
    return np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)


@pytest.mark.parametrize("periodic", [True, False])
def test_lattice_on_bin_edges(cuda, periodic):
    """separations exactly on the edges: bins are left-open, right-closed, on r"""
    pos = _lattice(8)
    for edges in ([1., 2., 3.], [0., 1., 2., 3.]):
        r, want = _run(pos, edges, [0, 1, 2], [8.] * 3, periodic)
        if periodic and edges[0] == 1.:
            # (1, 2]: r^2 = 2, 3, 4; (2, 3]: r^2 = 5, 6, 8, 9
            assert list(r.npairs) == [512 * 26, 512 * 90]
    _run(pos.astype("f4"), [0., 1., np.sqrt(2.), 2.], [0, 3], [8.] * 3, periodic)


@pytest.mark.parametrize("dtype", ["f4", "f8"])
def test_duplicates_and_box_faces(cuda, dtype):
    rng = np.random.RandomState(4)
    L = 20.
    pos = rng.uniform(size=(2000, 3)) * L
    pos[:40] = 0.
    pos[40:80, 0] = L
    pos[80:120, 1] = -1e-7
    pos[120:160, 2] = L + 1e-6
    pos[160:200] = -1e-9
    pos[200:260] = pos[260:320]                                # duplicates: r = 0 never counts
    pos = pos.astype(dtype)
    w = rng.uniform(0.5, 2., len(pos))
    _run(pos, [0., 1., 2.5, 4.], [0, 1, 2, 5], [L] * 3, True, w)
    _run(pos, [0., 1., 2.5, 4.], [0, 2], [L] * 3, False, w)


def test_empty_and_single_object(cuda):
    from nbodykit_b200.lab import SimulationBox3PCF
    edges = np.linspace(0., 5., 4)
    for n in (0, 1):
        pos = np.full((n, 3), 3.)
        for periodic in (True, False):
            r = SimulationBox3PCF(_cat(pos, np.ones(n), [20.] * 3), [0, 1], edges, periodic=periodic)
            assert (r.npairs == 0).all() and (r.poles["corr_0"] == 0).all() and (r.poles["corr_1"] == 0).all()
            assert r.poles.shape == (3, 3)


def test_permuted_input(cuda):
    from nbodykit_b200.lab import SimulationBox3PCF
    pos = to.clustered(8, 40., 2000, 3, 300, 0.6, dtype="f4")
    w = np.random.RandomState(9).uniform(-1., 2., len(pos))
    p = np.random.RandomState(10).permutation(len(pos))
    edges, poles = np.linspace(0., 5., 6), [0, 1, 4]
    r1 = SimulationBox3PCF(_cat(pos, w, [40.] * 3), poles, edges)
    r2 = SimulationBox3PCF(_cat(pos[p], w[p], [40.] * 3), poles, edges)
    np.testing.assert_array_equal(r1.npairs, r2.npairs)
    want = to.compute(pos, edges, poles, box=[40.] * 3, w=w)
    _within(_zeta(r1, poles), dict(zeta=_zeta(r2, poles), bound=want["bound"]), 1e-12)


def test_save_load_computed(cuda, tmp_path):
    from nbodykit_b200.lab import SimulationBox3PCF
    pos = np.random.RandomState(12).uniform(size=(1500, 3)) * 25.
    r = SimulationBox3PCF(_cat(pos, np.ones(len(pos)), [25.] * 3), [2, 0], np.linspace(0., 4., 5))
    f = str(tmp_path / "t.json")
    r.save(f)
    s = SimulationBox3PCF.load(f, comm=r.comm)
    np.testing.assert_array_equal(s.poles.data, r.poles.data)
    assert s.attrs["poles"] == [2, 0]


# ---- several ranks over gloo on device 0 -----------------------------------------------------------------------------
def _ranks(comm, pos, w, box, periodic, edges, poles, split):
    from nbodykit_b200.lab import ArrayCatalog, SimulationBox3PCF
    mine = slice(split[comm.rank], split[comm.rank + 1])
    data = {"Position": torch.from_numpy(np.ascontiguousarray(pos[mine])).cuda(),
            "Weight": torch.from_numpy(np.ascontiguousarray(w[mine])).cuda()}
    r = SimulationBox3PCF(ArrayCatalog(data, comm=comm, BoxSize=np.asarray(box, "f8")), poles, edges, periodic=periodic)
    return dict(npairs=r.npairs, zeta=np.stack([r.poles["corr_%d" % ell] for ell in poles]), cand=r.candidates)


_MULTI = [  # P, periodic, empty rank, slab-local rows
    (2, True, False, False),
    (3, True, True, True),
    (3, False, False, False),
    (2, False, True, True),
]


@pytest.mark.parametrize("case", range(len(_MULTI)))
def test_several_ranks_equal_one(cuda, case):
    from test_gpu_fof import _spawn
    from nbodykit_b200.lab import SimulationBox3PCF
    P, periodic, empty, local = _MULTI[case]
    L = 40.
    pos = to.clustered(20 + case, L, 2500, 3, 300, 0.7, dtype="f4")
    if local:
        pos = pos[np.argsort(pos[:, 0], kind="stable")]
    w = np.random.RandomState(case).uniform(-0.5, 2., len(pos))
    edges, poles = np.linspace(0., 6., 6), [0, 1, 2, 7]
    n = len(pos)
    split = [0, 0] + [n * (r + 1) // (P - 1) for r in range(P - 1)] if empty else [r * n // P for r in range(P + 1)]
    parts = _spawn(_ranks, P, pos, w, [L] * 3, periodic, edges, poles, split)
    one = SimulationBox3PCF(_cat(pos, w, [L] * 3), poles, edges, periodic=periodic)
    want = to.compute(pos, edges, poles, box=[L] * 3 if periodic else None, w=w)
    np.testing.assert_array_equal(one.npairs, want["npairs"])
    for p in parts:
        np.testing.assert_array_equal(p["npairs"], one.npairs)
        _within(p["zeta"], dict(zeta=_zeta(one, poles), bound=want["bound"]), 1e-12)
    assert want["npairs"].sum() > 10000


def test_two_gpu_threeptcf_matches_one_gpu():
    """launches tests/mgpu_check_threeptcf.py under torchrun when the box has >= 2 GPUs"""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29533", os.path.join(ROOT, "tests", "mgpu_check_threeptcf.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    sys.stdout.write(out.stdout[-3000:])
    sys.stderr.write(out.stderr[-3000:])
    assert out.returncode == 0
