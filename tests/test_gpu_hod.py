"""HaloCatalog.populate / repopulate on the GPU against the float64 restatement of oracle/hod_oracle.py: the same rows in
the same order (halo_id, gal_type and so the per-halo counts exactly), satellite positions and velocities to 1e-12 of
the column scale in float64 and within one float32 spacing of the cast float64 answer in float32, for the default and
the docs' parameters, modulate_with_cenocc on and off, mdef vir / 200c / 500m, a non-cubic box and a satellite-heavy
model that runs the PTRS sampler; periodic wrapping across every face; repopulate; P = 2 and 3 processes over gloo
sharing device 0 (one with no halos); and the reference's test_hod_cm / test_hod_peak flows through FOF.to_halos,
KDDensity, VectorProjection and FFTPower(mode='2d').  tests/mgpu_check_hod.py runs the several-rank comparison under
torchrun on several GPUs."""
import datetime
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import hod_oracle as ho

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Z = 0.55
DEFAULTS = dict(logMmin=12.02, sigma_logM=0.26, logM0=11.38, logM1=13.31, alpha=1.06)


def _cosmo():
    from nbodykit_b200.cosmology import Planck15
    return Planck15


def make_halos(n, seed, box, dtype="f8", lo=11., hi=15.5):
    rs = np.random.RandomState(seed)
    box = np.broadcast_to(np.asarray(box, "f8"), (3,))
    mass = 10 ** rs.uniform(lo, hi, n)
    pos = (rs.uniform(size=(n, 3)) * box).astype(dtype)
    vel = rs.normal(0, 300., size=(n, 3)).astype(dtype)
    return mass, pos, vel


def halo_catalog(mass, pos, vel, box, mdef="vir", comm=None, device=True):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ArrayCatalog, HaloCatalog
    conv = (lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()) if device else np.ascontiguousarray
    src = ArrayCatalog({"Mass": conv(mass), "Position": conv(pos), "Velocity": conv(vel)}, comm=comm or SelfComm(),
                       BoxSize=np.broadcast_to(np.asarray(box, "f8"), (3,)).copy())
    return HaloCatalog(src, _cosmo(), Z, mdef=mdef)


def oracle_for(halos, params, seed, modulate=True, h0=0):
    def host(name):
        v = halos[name].compute()
        return v.cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
    rsd = (1 + Z) / (100. * _cosmo().efunc(Z))
    return ho.populate(host("Mass"), host("Radius"), host("Concentration"), host("Position"), host("Velocity"),
                       halos.attrs["BoxSize"], params, seed, h0=h0, modulate=modulate, rsd=rsd)


def host_cols(cat):
    return {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v))
            for k, v in ((k, cat[k].compute()) for k in cat.columns if k not in ("Selection", "Weight", "Value"))}


def assert_matches(got, want, L):
    """rows identical; positions and velocities to 1e-12 of their scale (f8) or one float32 spacing (f4)"""
    np.testing.assert_array_equal(got["halo_id"], want["halo_id"])
    np.testing.assert_array_equal(got["gal_type"], want["gal_type"])
    for name, scale in (("Position", np.max(L)), ("Velocity", None), ("VelocityOffset", None)):
        a, b = got[name], want[name]
        assert a.dtype == b.dtype, name
        if a.dtype == np.float64:
            s = scale if scale is not None else max(1.0, np.abs(b).max())
            assert np.abs(a - b).max() <= 1e-12 * s, name
        else:
            d = np.abs(a.astype("f8") - b.astype("f8"))
            assert (d <= np.spacing(np.abs(b)).astype("f8") + 1e-30).all(), name
    np.testing.assert_allclose(got["host_centric_distance"], want["host_centric_distance"], rtol=1e-12, atol=1e-15)


CASES = [
    # params, modulate, mdef, dtype, box
    ({}, True, "vir", "f8", 1000.),
    (dict(alpha=0.5, sigma_logM=0.40), True, "200c", "f8", 1000.),
    ({}, False, "500m", "f8", [1000., 700., 1300.]),
    ({}, True, "vir", "f4", 1000.),
    (dict(alpha=0.5, sigma_logM=0.40), False, "200c", "f4", [1000., 700., 1300.]),
    (dict(logM1=12.5), True, "vir", "f8", 1000.),          # satellite-heavy: many PTRS draws
]


@pytest.mark.parametrize("params,modulate,mdef,dtype,box", CASES)
def test_against_oracle(cuda, params, modulate, mdef, dtype, box):
    from nbodykit_b200.lab import Zheng07Model
    mass, pos, vel = make_halos(200000, 3, box, dtype)
    halos = halo_catalog(mass, pos, vel, box, mdef)
    cat = halos.populate(Zheng07Model(modulate_with_cenocc=modulate), seed=1234, **params)
    p = dict(DEFAULTS, **params)
    want = oracle_for(halos, p, 1234, modulate)
    got = host_cols(cat)
    assert_matches(got, want, np.broadcast_to(box, (3,)))
    local = got["halo_id"]
    np.testing.assert_array_equal(got["halo_num_centrals"], want["ncen"][local])
    np.testing.assert_array_equal(got["halo_num_satellites"], want["nsat"][local])
    np.testing.assert_array_equal(got["halo_m" + mdef], mass[local])
    assert cat.csize == want["ncen"].sum() + want["nsat"].sum()
    assert cat.attrs["fsat"] == want["nsat"].sum() / cat.csize
    assert cat.attrs["gal_types"] == {"centrals": 0, "satellites": 1}
    assert cat.attrs["seed"] == 1234 and cat.attrs["alpha"] == p["alpha"]
    if "logM1" in params:
        lam = ho.mean_satellite(mass, **p)
        assert (lam >= 10).sum() > 1000 and want["nsat"].max() > 500


def test_wrapping_and_radius(cuda):
    """halos within 0.3 Mpc/h of every face of a 50 Mpc/h box: satellites cross each face and wrap into [0, L)"""
    from nbodykit_b200.lab import Zheng07Model
    rs = np.random.RandomState(9)
    n = 20000
    L = np.array([50., 40., 60.])
    mass = 10 ** rs.uniform(13.5, 15.0, n)
    pos = rs.uniform(size=(n, 3)) * L
    face = rs.randint(0, 6, n)
    for i in range(n):
        d = face[i] % 3
        pos[i, d] = rs.uniform(0, 0.3) if face[i] < 3 else L[d] - rs.uniform(0, 0.3)
    vel = np.zeros((n, 3))
    halos = halo_catalog(mass, pos, vel, L)
    cat = halos.populate(Zheng07Model, seed=5)
    got = host_cols(cat)
    want = oracle_for(halos, DEFAULTS, 5)
    assert_matches(got, want, L)
    p = got["Position"]
    assert (p >= 0).all() and (p < L).all()
    sat = got["gal_type"] == 1
    hp = pos[got["halo_id"][sat]]
    dx = p[sat] - hp
    for d in range(3):
        assert (dx[:, d] > L[d] / 2).sum() > 10 and (dx[:, d] < -L[d] / 2).sum() > 10
    R = halos["Radius"].compute().cpu().numpy()[got["halo_id"]]
    assert (got["host_centric_distance"] <= R).all()
    assert (got["host_centric_distance"][~sat] == 0).all()
    np.testing.assert_array_equal(got["halo_r" + "vir"], R)


def test_repopulate(cuda):
    from nbodykit_b200.lab import Zheng07Model
    mass, pos, vel = make_halos(50000, 4, 500.)
    halos = halo_catalog(mass, pos, vel, 500.)
    hod = halos.populate(Zheng07Model, seed=42)
    first = host_cols(hod)
    size = hod.csize
    hod.repopulate(seed=42)
    again = host_cols(hod)
    assert hod.csize == size
    for k in first:
        np.testing.assert_array_equal(first[k], again[k], err_msg=k)
    hod.repopulate(seed=None)
    assert isinstance(hod.attrs["seed"], int) and 0 <= hod.attrs["seed"] < 2 ** 32
    hod.repopulate(seed=42, alpha=1.0)
    assert hod.csize != size and hod.attrs["alpha"] == 1.0
    want = oracle_for(halos, dict(DEFAULTS, alpha=1.0), 42)
    assert_matches(host_cols(hod), want, np.full(3, 500.))
    with pytest.raises(ValueError):
        hod.repopulate(seed=42, bad_param_name=1.0)
    with pytest.raises(ValueError):
        halos.populate(Zheng07Model, seed=42, logMmin=17)
    assert halos.populate(Zheng07Model).attrs["seed"] is not None


def test_host_columns_and_overwritten_concentration(cuda):
    """host NumPy halo columns, float32 masses, and a user Concentration column"""
    from nbodykit_b200.lab import Zheng07Model
    mass, pos, vel = make_halos(30000, 6, 800.)
    halos = halo_catalog(mass.astype("f4"), pos, vel, 800., device=False)
    halos["Concentration"] = np.full(30000, 4.0)
    cat = halos.populate(Zheng07Model, seed=8)
    want = oracle_for(halos, DEFAULTS, 8)
    assert_matches(host_cols(cat), want, np.full(3, 800.))
    assert (host_cols(cat)["conc_NFWmodel"] == 4.0).all()


# ---- several ranks over gloo, sharing device 0

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


def _hod_ranks(comm, mass, pos, vel, box, split):
    from nbodykit_b200.lab import Zheng07Model
    mine = slice(split[comm.rank], split[comm.rank + 1])
    halos = halo_catalog(mass[mine], pos[mine], vel[mine], box, comm=comm)
    cat = halos.populate(Zheng07Model, seed=77)
    out = host_cols(cat)
    cat.repopulate(seed=78, alpha=0.8)
    out2 = host_cols(cat)
    return dict(first=out, second=out2, fsat=cat.attrs["fsat"], csize=cat.csize)


def _merged(parts):
    """the rows of all ranks in one rank's order: by (gal_type, halo_id), satellites of a halo in k order (stable)"""
    cols = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
    order = np.lexsort((cols["halo_id"], cols["gal_type"]))
    return {k: v[order] for k, v in cols.items()}


@pytest.mark.parametrize("P,split", [(2, [0, 0, 60000]), (3, [0, 25000, 25000, 60000])])
def test_several_ranks(cuda, P, split):
    from nbodykit_b200.lab import Zheng07Model
    mass, pos, vel = make_halos(60000, 11, 600.)
    res = _spawn(_hod_ranks, P, mass, pos, vel, 600., split)
    for key, seed, params in (("first", 77, DEFAULTS), ("second", 78, dict(DEFAULTS, alpha=0.8))):
        one = halo_catalog(mass, pos, vel, 600.).populate(Zheng07Model, seed=seed, **params)
        want = host_cols(one)
        got = _merged([r[key] for r in res])
        for k in want:
            np.testing.assert_array_equal(got[k], want[k], err_msg="%s %s" % (key, k))
    assert all(r["csize"] == res[0]["csize"] for r in res)
    assert all(r["fsat"] == res[0]["fsat"] for r in res)


# ---- the reference's test_hod_cm and test_hod_peak flows

@pytest.mark.parametrize("posdef", ["cm", "peak"])
def test_reference_flows(cuda, posdef):
    from nbodykit_b200 import transform
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.cosmology import NoWiggleEHPower
    from nbodykit_b200.lab import FFTPower, FOF, KDDensity, LogNormalCatalog, Zheng07Model
    cosmo = _cosmo()
    Plin = NoWiggleEHPower(redshift=Z)
    source = LogNormalCatalog(Plin=Plin, nbar=3e-3, BoxSize=512, Nmesh=128, seed=42, comm=SelfComm())
    if posdef == "peak":
        source["Density"] = KDDensity(source).density
    r = FOF(source, linking_length=0.2, nmin=20)
    halos = r.to_halos(cosmo=cosmo, redshift=Z, particle_mass=1e12, mdef="vir", posdef=posdef)
    assert halos.csize > 100 and halos.attrs["particle_mass"] == 1e12
    feats = r.find_features(peakcolumn="Density" if posdef == "peak" else None)
    length = np.asarray(feats["Length"].compute())
    keep = length > 0
    np.testing.assert_array_equal(np.asarray(halos["Mass"].compute()), 1e12 * length[keep])
    prefix = "CM" if posdef == "cm" else "Peak"
    np.testing.assert_array_equal(np.asarray(halos["Position"].compute()),
                                  np.asarray(feats[prefix + "Position"].compute())[keep])
    hod = halos.populate(Zheng07Model, seed=42)
    want = oracle_for(halos, DEFAULTS, 42)
    assert_matches(host_cols(hod), want, np.full(3, 512.))
    hod["Position"] += transform.VectorProjection(hod["VelocityOffset"], [0, 0, 1])
    p = FFTPower(hod.to_mesh(Nmesh=128), mode="2d", Nmu=5, los=[0, 0, 1])
    modes = np.asarray(p.power["modes"])
    assert modes.sum() > 0 and np.isfinite(np.asarray(p.power["power"])[modes > 0]).all()
