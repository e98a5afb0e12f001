"""Host-side checks of the Leauthaud11 and Hearin15 models (DESIGN.md 4.13) that need no GPU: the inverted Behroozi10
relation, the central occupation at the threshold, the package's spline against the oracle's, the assembly-bias
perturbation's bounds and bin average, percentile ties, the package's percentile stage on one rank, and every argument
error raised before any device work."""
import math

import numpy as np
import pytest
from scipy.interpolate import splev

from oracle import hod_models_oracle as hm
from oracle import zhist_oracle as zo


def _cosmo():
    from nbodykit_b200.cosmology import Planck15
    return Planck15


PARAM_SETS = [{}, dict(smhm_m1_0=12.6, smhm_beta_0=0.5, smhm_gamma_0=1.2), dict(smhm_delta_0=0.4, smhm_m0_a=0.2)]


@pytest.mark.parametrize("z", [0.0, 0.55, 1.2])
@pytest.mark.parametrize("extra", PARAM_SETS)
def test_inverse_reproduces_the_table(z, extra):
    from nbodykit_b200 import hod
    p = dict(hod.Leauthaud11Model(**extra).param_dict)
    t, c = hod.smhm_spline(p, z)
    logms = np.linspace(8.52, 12.48, 397)
    lmh = hod.behroozi10_log_mhalo(logms, p, z)
    assert np.abs(splev(lmh, (t, c, 3)) - logms).max() < 1e-6
    assert np.abs(zo.splev(lmh, t, c, 0)[0] - logms).max() < 1e-6


@pytest.mark.parametrize("z", [0.0, 0.55, 1.2])
@pytest.mark.parametrize("extra", PARAM_SETS)
def test_package_spline_is_the_oracles(z, extra):
    from nbodykit_b200 import hod
    p = dict(hod.Leauthaud11Model(**extra).param_dict)
    t, c = hod.smhm_spline(p, z)
    to, co = hm.spline(p, z)
    assert np.array_equal(t, to) and np.array_equal(c, co)
    assert np.array_equal(hod.behroozi10_log_mhalo(hod.SMHM_LOGMS, p, z), hm.log_mhalo(hm.LOGMS, p, z))
    occ = hod.Leauthaud11Model(threshold=10.2, **extra).occupation(z)
    assert (occ['Msat'], occ['Mcut']) == hm.sat_masses(p, z, 10.2)


def test_hand_values_at_z0():
    from nbodykit_b200.hod import Hearin15Model, Leauthaud11Model
    m = Leauthaud11Model()
    assert m.param_dict == hm.LEAUTHAUD11 and m.threshold == 10.5 and m.modulate_with_cenocc
    assert Hearin15Model().param_dict == hm.HEARIN15
    assert abs(float(hm.log_mhalo(10.5, hm.LEAUTHAUD11, 0.0)) - 11.534) < 5e-4
    msat, mcut = hm.sat_masses(hm.LEAUTHAUD11, 0.0)
    assert abs(msat / 4.23e12 - 1) < 2e-3 and abs(mcut / 1.69e12 - 1) < 3e-3
    assert abs(float(hm.mean_central(np.array([1e12]), hm.LEAUTHAUD11, 0.0)[0]) - 0.982) < 5e-4


def test_central_occupation_is_half_at_the_threshold():
    masses = 10 ** np.array([11.0, 11.7, 12.3, 13.5])
    for z in (0.0, 0.55):
        logms = hm.mean_log_mstar(masses, hm.LEAUTHAUD11, z)
        for m, thr in zip(masses, logms):
            assert hm.mean_central(np.array([m]), hm.LEAUTHAUD11, z, threshold=thr)[0] == 0.5
    # and at the halo mass of the threshold, to the accuracy of the inverse
    knee = 10 ** float(hm.log_mhalo(10.5, hm.LEAUTHAUD11, 0.55))
    assert abs(hm.mean_central(np.array([knee]), hm.LEAUTHAUD11, 0.55)[0] - 0.5) < 1e-5


@pytest.mark.parametrize("A", [-1.0, -0.3, 0.0, 0.5, 1.0])
@pytest.mark.parametrize("split", [0.25, 0.5, 0.75])
def test_perturbation_bounds_and_average(A, split):
    for hi, nb in ((1.0, np.linspace(0.0, 1.0, 1001)), (np.inf, np.concatenate([[0.0], np.geomspace(1e-8, 300., 1000)]))):
        up = hm.perturb(nb, A, split, hi, True)
        lo = hm.perturb(nb, A, split, hi, False)
        for v in (up, lo):
            assert (v >= 0).all() and (v <= hi).all()
        avg = (1 - split) * up + split * lo
        np.testing.assert_allclose(avg, nb, rtol=1e-13, atol=1e-15)
        if A == 0:
            assert np.array_equal(up, nb) and np.array_equal(lo, nb)
        elif A > 0:
            assert (up >= nb).all() and (lo <= nb).all()
        else:
            assert (up <= nb).all() and (lo >= nb).all()
    # the strength is clipped to [-1, 1]
    nb = np.linspace(0, 1, 11)
    assert np.array_equal(hm.perturb(nb, 3.0, split, 1.0, True), hm.perturb(nb, 1.0, split, 1.0, True))


def _bare_halos(mass, sec, h0=0):
    """a _Halos with just the columns the percentile stage reads, on the host, for one rank"""
    import torch
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.source.catalog.halos import _Halos
    h = _Halos.__new__(_Halos)
    h.comm, h.n, h.h0 = SelfComm(), len(mass), h0
    h.mass = torch.as_tensor(np.asarray(mass, "f8"))
    h.sec = {"s": torch.as_tensor(np.asarray(sec, "f8"))}
    h._pct = {}
    return h


def test_percentile_ties_by_global_row():
    # two bins of 0.5 dex: the first holds rows 0, 2, 3, 5 (sec 1, 1, 0, 1), the second rows 1, 4 (sec 2, 2)
    mass = 10 ** np.array([12.1, 12.6, 12.2, 12.3, 12.7, 12.05])
    sec = np.array([1.0, 2.0, 1.0, 0.0, 2.0, 1.0])
    want = np.array([2 / 4, 1 / 2, 3 / 4, 1 / 4, 2 / 2, 4 / 4])
    np.testing.assert_array_equal(hm.percentiles(mass, sec, 0.5), want)
    h = _bare_halos(mass, sec)
    np.testing.assert_array_equal(h.percentiles("s", 0.5).numpy(), want)
    assert ("s", 0.5) in h._pct
    # -0.0 and 0.0 tie
    sec0 = np.array([0.0, 0.0, -0.0, 0.0, 0.0, 0.0])
    np.testing.assert_array_equal(hm.percentiles(mass, sec0, 0.5), [1 / 4, 1 / 2, 2 / 4, 3 / 4, 2 / 2, 4 / 4])


def test_package_percentiles_are_the_oracles():
    rs = np.random.RandomState(4)
    mass = 10 ** rs.uniform(11, 15, 20000)
    sec = np.round(rs.uniform(2, 12, 20000), 1)        # many ties
    for d in (0.1, 0.37, 1.0):
        np.testing.assert_array_equal(_bare_halos(mass, sec).percentiles("s", d).numpy(),
                                      hm.percentiles(mass, sec, d))
    with pytest.raises(ValueError, match="mass bins"):
        _bare_halos(mass, sec).percentiles("s", 1e-9)


# ---- errors before any device work -----------------------------------------------------------------------------------------

def _halos(n=100, **kw):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ArrayCatalog, HaloCatalog
    rs = np.random.RandomState(1)
    cols = dict(Mass=10 ** rs.uniform(12, 14, n), Position=rs.uniform(0, 100, (n, 3)), Velocity=np.zeros((n, 3)))
    cols.update(kw)
    return HaloCatalog(ArrayCatalog(cols, comm=SelfComm(), BoxSize=100.), _cosmo(), 0.5)


def test_argument_errors_before_device_work(monkeypatch):
    from nbodykit_b200 import hod
    from nbodykit_b200.lab import Hearin15Model, Leauthaud11Model
    from nbodykit_b200.source.catalog import halos as H

    def no_device(*a, **k):
        raise AssertionError("device work before the argument checks")
    monkeypatch.setattr(H._Halos, "run", no_device)
    monkeypatch.setattr(H._Halos, "percentiles", no_device)
    halos = _halos()
    for model in (Leauthaud11Model, Hearin15Model):
        with pytest.raises(ValueError, match="invalid"):
            halos.populate(model, seed=1, logMmin=12.)
        with pytest.raises(ValueError, match="invalid"):
            model(bad_param=1.)
        with pytest.raises(ValueError, match="scatter"):
            halos.populate(model, seed=1, scatter_model_param1=0.)
        with pytest.raises(ValueError, match="finite"):
            halos.populate(model, seed=1, bsat=np.nan)
        with pytest.raises(ValueError, match="finite"):
            halos.populate(model(threshold=np.inf), seed=1)
        with pytest.raises(ValueError, match="bsat"):
            halos.populate(model, seed=1, bsat=-1.)
        with pytest.raises(ValueError, match="increasing"):
            halos.populate(model, seed=1, smhm_beta_0=-3.)
        with pytest.raises(ValueError, match="seed"):
            halos.populate(model, seed=-1)
        with pytest.raises(NotImplementedError, match="halotools"):
            model.to_halotools(_cosmo(), 0.5, "vir")
    for split in (0., 1., -0.5, 1.5, np.nan):
        with pytest.raises(ValueError, match="split"):
            halos.populate(Hearin15Model(split=split), seed=1)
    for d in (0., -0.1, np.inf, np.nan):
        with pytest.raises(ValueError, match="dlog10_prim_haloprop"):
            halos.populate(Hearin15Model(dlog10_prim_haloprop=d), seed=1)
    with pytest.raises(ValueError, match="no sec_haloprop column 'Spin'"):
        halos.populate(Hearin15Model(sec_haloprop="Spin"), seed=1)
    for v in (np.nan, np.inf, -np.inf):
        bad = _halos()
        arr = np.linspace(0.1, 1.0, 100)
        arr[17] = v
        bad["Spin"] = arr
        with pytest.raises(ValueError, match="non-finite"):
            bad.populate(Hearin15Model(sec_haloprop="Spin"), seed=1)
    bad = _halos()
    bad["Spin"] = np.ones((100, 2))
    with pytest.raises(ValueError, match="one-dimensional"):
        bad.populate(Hearin15Model(sec_haloprop="Spin"), seed=1)

    class Other(hod.HODModel):      # an HODModel the package does not implement
        pass
    with pytest.raises(NotImplementedError, match="Leauthaud11Model"):
        halos.populate(Other, seed=1)


def test_models_and_exports():
    import nbodykit_b200.hod as hod
    import nbodykit_b200.lab as lab
    from nbodykit_b200.hod import HODModel, Hearin15Model, Leauthaud11Model
    assert lab.Leauthaud11Model is Leauthaud11Model and lab.Hearin15Model is Hearin15Model
    assert set(hod.__all__) == {"HODModel", "Zheng07Model", "Leauthaud11Model", "Hearin15Model"}
    assert issubclass(Leauthaud11Model, HODModel) and issubclass(Hearin15Model, Leauthaud11Model)
    m = Hearin15Model(threshold=10.8, modulate_with_cenocc=False, sec_haloprop="Spin", split=0.3,
                      dlog10_prim_haloprop=0.2, alphasat=1.1)
    assert m.arguments() == dict(threshold=10.8, modulate_with_cenocc=False, sec_haloprop="Spin", split=0.3,
                                 dlog10_prim_haloprop=0.2)
    assert m.param_dict["alphasat"] == 1.1
    m.update(dict(mean_occupation_centrals_assembias_param1=-4., mean_occupation_satellites_assembias_param1=0.4))
    assert m.strengths() == (-1.0, 0.4)
    from nbodykit_b200.source.catalog.halos import _as_model
    c = _as_model(m)
    assert type(c) is Hearin15Model and c is not m
    assert c.arguments() == m.arguments() and c.param_dict == m.param_dict
    c = _as_model(Leauthaud11Model)
    assert type(c) is Leauthaud11Model and c.threshold == 10.5
    assert math.isfinite(c.occupation(0.55)["Msat"])
