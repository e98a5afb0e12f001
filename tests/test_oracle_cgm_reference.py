"""oracle/cgm_oracle.py pinned against the reference's own cylinder grouping: `cgm()` of nbodykit/algorithms/cgm.py run
verbatim on one rank (oracle/cgm_refload.py) and `direct_cgm` of its tests, on the reference tests' catalogues.  The
golden fixtures store the reference's output for the GPU tests.  Skipped where the reference tree is absent."""
import os

import numpy as np
import pytest

from oracle import cgm_oracle as co, cgm_refload

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.skipif(not cgm_refload.available(), reason="reference tree not present")


def _reference_catalogue(seed=42, L=256.):
    """the catalogue of the reference's test_periodic_cgm / test_nonperiodic_cgm, drawn with NumPy"""
    rng = np.random.RandomState(seed)
    n = int(3e-4 * L ** 3)
    pos = rng.uniform(size=(n, 3)) * L
    logm = rng.uniform(12, 15, size=n)
    gal = np.empty(n)
    gal[logm < 14.5] = 0
    gal[logm > 14.5] = 1
    return pos, 10 ** logm, gal


@pytest.mark.parametrize("periodic", [True, False])
def test_oracle_equals_reference_cgm_and_direct_cgm(periodic):
    ref = cgm_refload.load()
    pos, mass, gal = _reference_catalogue()
    t, h, s, prio = co.cgm(pos, [mass, gal], 10., 10., los=[0, 0, 1], periodic=periodic, BoxSize=256.)
    rt, rh, rs = cgm_refload.run_cgm(pos, prio, 10., 10., np.array([0., 0., 1.]),
                                     np.array([256.] * 3) if periodic else None)
    dn, dt, dh = ref.direct_cgm(pos, mass, gal, 10., 10., periodic=periodic, BoxSize=[256.] * 3)
    for mine, theirs, direct in ((t, rt, dt), (h, rh, dh), (s, rs, dn)):
        np.testing.assert_array_equal(mine, theirs)
        np.testing.assert_array_equal(mine, direct)
    assert (t == 1).sum() > 100


def test_oracle_equals_reference_cgm_observer_at_origin():
    rng = np.random.RandomState(1)
    n = 3000
    u = rng.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1)[:, None]
    pos = u * rng.uniform(100., 120., size=n)[:, None]
    t, h, s, prio = co.cgm(pos, [rng.uniform(size=n)], 5., 12.)
    for mine, theirs in zip((t, h, s), cgm_refload.run_cgm(pos, prio, 5., 12., None, None)):
        np.testing.assert_array_equal(mine, theirs)


def test_golden_fixtures_hold_the_reference_output():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_cgm_golden", os.path.join(ROOT, "tests", "golden", "make_cgm_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    for name, (pos, mass, gal, rperp, rpar, los, periodic, L) in mk.cases().items():
        z = np.load(os.path.join(ROOT, "tests", "golden", "cgm_%s.npz" % name))
        np.testing.assert_array_equal(z["pos"], pos)
        prio = co.priority([mass, gal], len(pos))
        got = cgm_refload.run_cgm(pos, prio, rperp, rpar, los, np.array([L] * 3) if periodic else None)
        for c, g in zip(("cgm_type", "cgm_haloid", "num_cgm_sats"), got):
            np.testing.assert_array_equal(z[c], g)


def test_priority_matches_lexsort_with_ties_by_row():
    rng = np.random.RandomState(2)
    a = rng.randint(0, 3, size=500)
    b = np.where(rng.uniform(size=500) < 0.5, -0.0, 0.0)
    prio = co.priority([a, b], 500)
    order = np.lexsort((np.arange(500), a))
    np.testing.assert_array_equal(np.argsort(prio), order)
