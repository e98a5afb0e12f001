"""oracle/kddensity_oracle.py pinned against the reference's own KDDensity (nbodykit/algorithms/kdtree.py run verbatim
on one rank by oracle/kddensity_refload.py), bit for bit, on uniform and clustered float32 / float64 catalogues; the
contract's distance checked against brute force; the golden fixtures hold the reference's output.  Skipped where the
reference tree is absent."""
import os
import warnings

import numpy as np
import pytest

from oracle import kddensity_oracle as ko, kddensity_refload

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.skipif(not kddensity_refload.available(), reason="reference tree not present")


def _catalogue(kind, dtype, n=3000, L=64., seed=1):
    rng = np.random.RandomState(seed)
    if kind == "uniform":
        pos = rng.uniform(size=(n, 3)) * L
    else:
        centres = rng.uniform(size=(20, 3)) * L
        pos = np.concatenate([rng.uniform(size=(n // 3, 3)) * L,
                              (centres[rng.randint(0, 20, n - n // 3)] + rng.normal(scale=0.5, size=(n - n // 3, 3))) % L])
    return pos.astype(dtype), L


@pytest.mark.parametrize("kind", ["uniform", "clustered"])
@pytest.mark.parametrize("dtype", ["f4", "f8"])
def test_oracle_equals_reference(kind, dtype):
    pos, L = _catalogue(kind, dtype)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref, attrs = kddensity_refload.run(pos, L)
        _, mine = ko.density(pos, L)
    np.testing.assert_array_equal(mine, ref)
    np.testing.assert_array_equal(attrs["BoxSize"], [L] * 3)
    assert attrs["meansep"] == (len(pos) / L ** 3) ** (1 / 3.) and attrs["margin"] == 1.0


@pytest.mark.parametrize("dtype", ["f4", "f8"])
def test_distance_is_the_contract_restated(dtype):
    """the 8th smallest of sqrt((dx^2 + dy^2) + dz^2) with the per-axis wrap, in float64, equals cKDTree's"""
    pos, L = _catalogue("clustered", dtype, n=600, seed=2)
    q = ko.unit(pos, L).astype("f8")
    dx = q[:, None, :] - q[None, :, :]
    dx = np.where(dx > 0.5, dx - 1, np.where(dx < -0.5, dx + 1, dx))
    d = np.sqrt((dx[..., 0] * dx[..., 0] + dx[..., 1] * dx[..., 1]) + dx[..., 2] * dx[..., 2])
    np.testing.assert_array_equal(np.sort(d, axis=1)[:, ko.K - 1], ko.distance(pos, L))


def test_unit_coordinates_rounding_to_one_become_zero():
    pos = np.array([[-1e-7, 0., 63.99999], [64., -64., 128.5]], dtype="f4")
    q = ko.unit(pos, 64.)
    assert q.dtype == np.float32 and (q >= 0).all() and (q < 1).all()
    assert q[0, 0] == 0.0 and q[1, 0] == 0.0 and q[1, 1] == 0.0


def test_golden_fixtures_hold_the_reference_output():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_kddensity_golden",
                                                  os.path.join(ROOT, "tests", "golden", "make_kddensity_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    for name, (pos, L) in mk.cases().items():
        z = np.load(os.path.join(ROOT, "tests", "golden", "kddensity_%s.npz" % name))
        np.testing.assert_array_equal(z["pos"], pos)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            np.testing.assert_array_equal(z["density"], kddensity_refload.run(pos, L)[0])
