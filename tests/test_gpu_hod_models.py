"""HaloCatalog.populate / repopulate with Leauthaud11Model and Hearin15Model on the GPU against the float64 restatement of
oracle/hod_models_oracle.py: the same rows (so the per-halo counts exactly), positions and velocities to 1e-12 in float64
and within one float32 spacing in float32, at several redshifts, thresholds, splits, strengths and bin widths and for a
user secondary property with ties; Hearin15 with zero strengths is Leauthaud11 bit for bit; the central occupation of the
upper and lower halves of every mass bin of 10^6 halos matches the perturbed means; repopulate equals a fresh populate;
and P = 2 and 3 processes over gloo sharing device 0 (one with no halos) equal P = 1 bit for bit, which needs the
percentiles to be ranked over all ranks.  tests/mgpu_check_hod_models.py runs the several-rank comparison under
torchrun on several GPUs."""
import math

import numpy as np
import pytest
import torch

from oracle import hod_models_oracle as hm
from test_gpu_hod import _merged, _spawn, assert_matches, host_cols, make_halos

pytestmark = pytest.mark.gpu


def _cosmo():
    from nbodykit_b200.cosmology import Planck15
    return Planck15


def halo_catalog(mass, pos, vel, box, z, comm=None, **extra):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ArrayCatalog, HaloCatalog

    def dev(a):
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()
    src = ArrayCatalog({"Mass": dev(mass), "Position": dev(pos), "Velocity": dev(vel)}, comm=comm or SelfComm(),
                       BoxSize=np.broadcast_to(np.asarray(box, "f8"), (3,)).copy())
    halos = HaloCatalog(src, _cosmo(), z)
    for k, v in extra.items():          # extra halo columns, or ones that overwrite Concentration
        halos[k] = dev(v)
    return halos


def _host(halos, name):
    v = halos[name].compute()
    return v.cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)


def oracle_for(halos, model, seed):
    """the oracle's catalogue of `model` (an instance) on the one-rank catalogue `halos`"""
    from nbodykit_b200.hod import Hearin15Model
    z = halos.attrs["redshift"]
    mass = _host(halos, "Mass").astype("f8")
    pct, split = None, 0.5
    if isinstance(model, Hearin15Model):
        pct = hm.percentiles(mass, _host(halos, model.sec_haloprop), model.dlog10_prim_haloprop)
        split = model.split
    rsd = (1 + z) / (100. * _cosmo().efunc(z))
    return hm.populate(mass, _host(halos, "Radius"), _host(halos, "Concentration"), _host(halos, "Position"),
                       _host(halos, "Velocity"), halos.attrs["BoxSize"], model.param_dict, seed, z,
                       threshold=model.threshold, modulate=model.modulate_with_cenocc, rsd=rsd, pct=pct, split=split)


def _model(name, args, params):
    from nbodykit_b200.lab import Hearin15Model, Leauthaud11Model
    cls = {"leauthaud11": Leauthaud11Model, "hearin15": Hearin15Model}[name]
    return cls(**args, **params)


CASES = [
    # model, constructor arguments, parameters, position dtype, redshift
    ("leauthaud11", {}, {}, "f8", 0.55),
    ("leauthaud11", dict(threshold=10.8, modulate_with_cenocc=False), dict(alphasat=1.2, bsat=6.0), "f4", 0.0),
    ("hearin15", {}, {}, "f8", 0.55),
    ("hearin15", dict(split=0.3, dlog10_prim_haloprop=0.2),
     dict(mean_occupation_centrals_assembias_param1=-0.6, mean_occupation_satellites_assembias_param1=0.9), "f4", 0.0),
    ("hearin15", dict(split=0.75, dlog10_prim_haloprop=0.05, threshold=10.2),
     dict(mean_occupation_centrals_assembias_param1=0.4, mean_occupation_satellites_assembias_param1=-1.0), "f8", 0.0),
]


@pytest.mark.parametrize("name,args,params,dtype,z", CASES)
def test_against_oracle(cuda, name, args, params, dtype, z):
    mass, pos, vel = make_halos(200000, 3, 1000., dtype, hi=14.8)
    halos = halo_catalog(mass, pos, vel, 1000., z)
    model = _model(name, args, params)
    cat = halos.populate(model, seed=1234)
    want = oracle_for(halos, model, 1234)
    got = host_cols(cat)
    assert_matches(got, want, np.full(3, 1000.))
    local = got["halo_id"]
    np.testing.assert_array_equal(got["halo_num_centrals"], want["ncen"][local])
    np.testing.assert_array_equal(got["halo_num_satellites"], want["nsat"][local])
    assert cat.csize == want["ncen"].sum() + want["nsat"].sum()
    assert want["ncen"].sum() > 10000 and want["nsat"].sum() > 1000
    assert cat.attrs["fsat"] == want["nsat"].sum() / cat.csize
    for k, v in model.arguments().items():
        assert cat.attrs[k] == v, k
    for k, v in model.param_dict.items():
        assert cat.attrs[k] == v, k


def test_user_secondary_property_with_ties(cuda):
    """a user column as sec_haloprop, with many ties (broken by global row) and negative zeros"""
    from nbodykit_b200.lab import Hearin15Model
    mass, pos, vel = make_halos(100000, 8, 700., hi=14.8)
    spin = np.round(np.random.RandomState(2).normal(0, 1, mass.size), 1)
    spin[spin == 0] = -0.0
    halos = halo_catalog(mass, pos, vel, 700., 0.3, Spin=spin)
    model = Hearin15Model(sec_haloprop="Spin", split=0.4)
    got = host_cols(halos.populate(model, seed=5))
    assert_matches(got, oracle_for(halos, model, 5), np.full(3, 700.))


@pytest.mark.parametrize("dtype", ["f4", "f8"])
def test_zero_strengths_is_leauthaud11(cuda, dtype):
    from nbodykit_b200.lab import Hearin15Model, Leauthaud11Model
    mass, pos, vel = make_halos(100000, 6, 500., dtype, hi=14.8)
    halos = halo_catalog(mass, pos, vel, 500., 0.55)
    a = host_cols(halos.populate(Leauthaud11Model, seed=17))
    b = host_cols(halos.populate(Hearin15Model, seed=17, mean_occupation_centrals_assembias_param1=0.,
                                 mean_occupation_satellites_assembias_param1=0.))
    assert a.keys() == b.keys()
    for k in a:
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def test_assembly_bias_statistics(cuda):
    """on 10^6 halos, the number of centrals in the upper and in the lower halos of every mass bin is the sum of their
    perturbed means within 5 sigma, and both differ from the unperturbed means"""
    from nbodykit_b200.lab import Hearin15Model
    n = 1000000
    rs = np.random.RandomState(12)
    mass = 10 ** rs.uniform(11.0, 12.6, n)
    pos = rs.uniform(0, 1000., (n, 3))
    vel = np.zeros((n, 3))
    conc = np.exp(rs.normal(2.0, 0.3, n))
    halos = halo_catalog(mass, pos, vel, 1000., 0.55, Concentration=conc)
    A, split, d = 0.5, 0.5, 0.1
    model = Hearin15Model(split=split, dlog10_prim_haloprop=d, mean_occupation_centrals_assembias_param1=A)
    got = host_cols(halos.populate(model, seed=99))
    ncen = np.zeros(n)
    ncen[got["halo_id"][got["gal_type"] == 0]] = 1
    pct = hm.percentiles(mass, conc, d)
    base, _ = hm.means(mass, model.param_dict, 0.55, pct=None)
    upper = pct > split
    pert = hm.perturb(base, A, split, 1.0, upper)
    b = np.floor(np.log10(mass) / d)
    checked = shifted = 0
    for v in np.unique(b):
        for half in (upper, ~upper):
            sel = (b == v) & half
            if sel.sum() < 1000:
                continue
            want = pert[sel].sum()
            sig = math.sqrt((pert[sel] * (1 - pert[sel])).sum())
            assert abs(ncen[sel].sum() - want) <= 5 * sig + 1e-9, (v, ncen[sel].sum(), want, sig)
            checked += 1
            shifted += abs(ncen[sel].sum() - base[sel].sum()) > 5 * sig
    assert checked >= 20 and shifted >= checked // 2


@pytest.mark.parametrize("name", ["leauthaud11", "hearin15"])
def test_repopulate_equals_populate(cuda, name):
    mass, pos, vel = make_halos(80000, 4, 500., hi=14.8)
    halos = halo_catalog(mass, pos, vel, 500., 0.55)
    model = _model(name, {}, {})
    hod = halos.populate(model, seed=42)
    new = dict(bsat=5.0, smhm_m1_0=12.2)
    if name == "hearin15":
        new.update(mean_occupation_centrals_assembias_param1=-0.5, mean_occupation_satellites_assembias_param1=0.7)
    hod.repopulate(seed=43, **new)
    again = host_cols(hod)
    fresh = host_cols(halos.populate(_model(name, {}, new), seed=43))
    assert again.keys() == fresh.keys()
    for k in fresh:
        np.testing.assert_array_equal(again[k], fresh[k], err_msg=k)
    assert hod.attrs["bsat"] == 5.0 and hod.attrs["seed"] == 43 and type(hod.model) is type(model)
    assert_matches(again, oracle_for(halos, _model(name, {}, new), 43), np.full(3, 500.))


# ---- several ranks over gloo, sharing device 0

MODEL_ARGS = dict(split=0.4, dlog10_prim_haloprop=0.15)


def _hod_ranks(comm, mass, pos, vel, box, split):
    from nbodykit_b200.lab import Hearin15Model
    mine = slice(split[comm.rank], split[comm.rank + 1])
    halos = halo_catalog(mass[mine], pos[mine], vel[mine], box, 0.55, comm=comm)
    cat = halos.populate(Hearin15Model(**MODEL_ARGS), seed=77)
    out = host_cols(cat)
    cat.repopulate(seed=78, mean_occupation_satellites_assembias_param1=-0.8)
    out2 = host_cols(cat)
    return dict(first=out, second=out2, fsat=cat.attrs["fsat"], csize=cat.csize)


@pytest.mark.parametrize("P,split", [(2, [0, 0, 60000]), (3, [0, 25000, 25000, 60000])])
def test_several_ranks(cuda, P, split):
    from nbodykit_b200.lab import Hearin15Model
    mass, pos, vel = make_halos(60000, 11, 600., hi=14.8)
    res = _spawn(_hod_ranks, P, mass, pos, vel, 600., split)
    for key, seed, params in (("first", 77, {}), ("second", 78, dict(mean_occupation_satellites_assembias_param1=-0.8))):
        one = halo_catalog(mass, pos, vel, 600., 0.55).populate(Hearin15Model(**MODEL_ARGS, **params), seed=seed)
        want = host_cols(one)
        got = _merged([r[key] for r in res])
        for k in want:
            np.testing.assert_array_equal(got[k], want[k], err_msg="%s %s" % (key, k))
    assert all(r["csize"] == res[0]["csize"] for r in res)
    assert all(r["fsat"] == res[0]["fsat"] for r in res)
