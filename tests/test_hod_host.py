"""Host-side checks of the HOD population (DESIGN.md 4.13) that need no GPU: the background quantities and halo relations
against hand-evaluated closed forms, the oracle's NFW radius inverse and Jeans integral against mpmath, the oracle's
samplers against the model's distributions, and every argument error raised before any device work."""
import math

import mpmath
import numpy as np
import pytest
from scipy import stats

from oracle import hod_oracle as ho

DEFAULTS = dict(logMmin=12.02, sigma_logM=0.26, logM0=11.38, logM1=13.31, alpha=1.06)


def _cosmo():
    from nbodykit_b200.cosmology import Planck15
    return Planck15


# ---- background quantities and halo relations -----------------------------------------------------------------------------

@pytest.mark.parametrize("z", [0.0, 0.55])
def test_omega_m_and_rho_crit(z):
    import torch
    c = _cosmo()
    E2 = c.efunc(z) ** 2
    assert abs(c.Omega_m(z) - c.Omega0_m * (1 + z) ** 3 / E2) <= 1e-15
    G = 6.67430e-11
    msun = 1.3271244e20 / G
    mpc = 3.0856775814913673e22
    H = 100e3 / mpc                                        # h s^-1
    rho = 3 * H ** 2 / (8 * math.pi * G) * mpc ** 3 / msun / 1e10 * E2
    assert abs(c.rho_crit(z) / rho - 1) < 1e-13
    t = torch.tensor([z, z], dtype=torch.float64)
    np.testing.assert_allclose(c.rho_crit(t).numpy(), [rho, rho], rtol=1e-13)
    np.testing.assert_allclose(c.Omega_m(np.array([z])), [c.Omega_m(z)], rtol=1e-15)


@pytest.mark.parametrize("z", [0.0, 0.55])
@pytest.mark.parametrize("mdef", ["vir", "200c", "500m"])
def test_halo_radius_and_concentration(z, mdef):
    from nbodykit_b200 import transform
    c = _cosmo()
    m = np.array([1e11, 1e12, 3e13, 1e15])
    rho_c = 27.75366272458308 * float(c.efunc(z)) ** 2 * 1e10
    om = c.Omega0_m * (1 + z) ** 3 / float(c.efunc(z)) ** 2
    if mdef == "vir":
        x = om - 1
        thr = (18 * math.pi ** 2 + 82 * x - 39 * x * x) * rho_c
    elif mdef == "200c":
        thr = 200 * rho_c
    else:
        thr = 500 * om * rho_c
    np.testing.assert_allclose(transform.HaloRadius(m, c, z, mdef), (3 * m / (4 * math.pi * thr)) ** (1 / 3.), rtol=1e-12)
    a = 0.537 + (1.025 - 0.537) * math.exp(-0.718 * z ** 1.08)
    b = -0.097 + 0.024 * z
    np.testing.assert_allclose(transform.HaloConcentration(m, c, z, mdef), 10 ** (a + b * np.log10(m / 1e12)), rtol=1e-13)
    np.testing.assert_allclose(transform.HaloVelocityDispersion(m, c, z),
                               1100. * (float(c.efunc(z)) * m / 1e15) ** 0.33333, rtol=1e-13)


def test_halo_relations_errors_and_kinds():
    import torch
    from nbodykit_b200 import transform
    from nbodykit_b200.base.catalog import Column
    c = _cosmo()
    for bad in ("200", "vir2", "0c", "200x", None):
        with pytest.raises(ValueError):
            transform.HaloRadius(np.ones(2) * 1e12, c, 0.5, bad)
    assert isinstance(transform.HaloRadius(torch.ones(2) * 1e12, c, 0.5), torch.Tensor)
    assert isinstance(transform.HaloConcentration(Column(np.ones(2) * 1e12), c, 0.5), Column)
    v = np.array([[1., 2., 3.], [-1., 0., 4.]])
    np.testing.assert_allclose(transform.VectorProjection(v, [0, 0, 2]), [[0, 0, 3], [0, 0, 4]])
    d = np.array([1., 1., 0.]) / 2 ** 0.5
    np.testing.assert_allclose(transform.VectorProjection(v, [1, 1, 0]), (v @ d)[:, None] * d[None, :], rtol=1e-15)


# ---- the oracle's NFW radius inverse and Jeans integral ---------------------------------------------------------------------

def test_nfw_inverse_against_mpmath():
    mpmath.mp.dps = 40
    worst = 0.
    for c in (1., 2.5, 7.3, 30., 100.):
        gc = mpmath.log(1 + c) - c / (1 + mpmath.mpf(c))
        for u in (1e-12, 1e-9, 1e-6, 1e-3, 0.05, 0.3, 0.5, 0.8, 0.99, 1 - 1e-6, 1 - 1e-12):
            y = float(ho.ginv(np.array(u) * ho.g(np.array(c))))
            want = -1 - 1 / mpmath.lambertw(-mpmath.exp(-1 - mpmath.mpf(u) * gc), 0)
            worst = max(worst, abs(y / float(want.real) - 1))
    assert worst < 1e-10, worst


def test_jeans_integral_against_mpmath():
    mpmath.mp.dps = 30

    def gm(t):
        return mpmath.log(1 + t) - t / (1 + t)
    worst = 0.
    for y in np.geomspace(1e-6, 100, 29):
        want = mpmath.quad(lambda t: gm(t) / (t ** 3 * (1 + t) ** 2), [y, 2 * y, 10 * y, 100 * y, mpmath.inf])
        worst = max(worst, abs(float(ho.jeans_integral(np.array(y))) / float(want) - 1))
    assert worst < 1e-9, worst
    s = ho.sigma_r2_over_v2(np.array([1e-300, 1e-30, 1e-12]), np.array(5.))
    assert np.isfinite(s).all() and (s >= 0).all() and s[-1] < 1e-9


def test_package_jeans_table_is_the_oracles():
    from nbodykit_b200 import hod
    assert np.array_equal(hod.jeans_table(), ho.jeans_table())
    assert (hod.JEANS_S0, hod.JEANS_HS, hod.JEANS_K) == (ho.S0, ho.HS, ho.K)


# ---- the oracle's samplers ---------------------------------------------------------------------------------------------

def test_mean_occupations():
    n = 200000
    for logm in (11.6, 11.9, 12.02, 12.2, 12.6, 13.5, 14.5):
        m = np.full(n, 10 ** logm)
        ncen, nsat = ho.occupy(m, 1000 * int(logm * 10), DEFAULTS, 7)
        pc = ho.mean_central(m[:1], DEFAULTS["logMmin"], DEFAULTS["sigma_logM"])[0]
        assert abs(ncen.mean() - pc) <= 5 * math.sqrt(pc * (1 - pc) / n) + 1e-12
        lam = ho.mean_satellite(m[:1], **DEFAULTS)[0]
        assert abs(nsat.mean() - lam) <= 5 * math.sqrt(lam / n) + 1e-12


@pytest.mark.parametrize("lam", [0.01, 0.5, 3., 12., 80., 1000.])
def test_poisson_chi2(lam):
    n = 200000
    k = ho.key(99, 0, np.arange(n))
    x = ho.poisson(k, np.full(n, lam))
    lo, hi = stats.poisson.ppf([1e-4, 1 - 1e-4], lam).astype(int)
    edges = np.arange(max(lo, 0), hi + 2)
    obs = np.array([(x < edges[1]).sum()] + [(x == e).sum() for e in edges[1:-2]] + [(x >= edges[-2]).sum()])
    p = np.concatenate([[stats.poisson.cdf(edges[0], lam)], stats.poisson.pmf(edges[1:-2], lam),
                        [stats.poisson.sf(edges[-2] - 1, lam)]])
    keep = p * n >= 5
    obs = np.concatenate([obs[keep], [obs[~keep].sum()]])
    exp = np.concatenate([p[keep], [p[~keep].sum()]]) * n
    obs, exp = obs[exp > 0], exp[exp > 0]
    chi2 = ((obs - exp) ** 2 / exp).sum()
    assert stats.chi2.sf(chi2, len(obs) - 1) > 1e-4, (chi2, len(obs))


def _satellites(n, c, seed=3):
    mass = np.full(n, 1e14)
    params = dict(DEFAULTS, logM0=0.0, logM1=14.0 - math.log10(5.0), alpha=1.0, sigma_logM=0.01, logMmin=10.)
    out = ho.populate(mass, np.full(n, 1.0), np.full(n, c), np.full((n, 3), 50.), np.zeros((n, 3)), 100., params, seed)
    return out, mass


@pytest.mark.parametrize("c", [2.0, 9.0, 40.0])
def test_radial_ks_against_nfw(c):
    out, _ = _satellites(20000, c)
    x = out["host_centric_distance"][out["gal_type"] == 1]
    assert x.size > 50000

    def cdf(r):
        return ho.g(c * np.asarray(r)) / ho.g(np.array(c))
    assert stats.kstest(x, cdf).pvalue > 1e-4


def test_velocity_dispersion_bins():
    c = 6.0
    out, mass = _satellites(20000, c, seed=4)
    sat = out["gal_type"] == 1
    x = out["host_centric_distance"][sat]
    v = out["Velocity"][sat]
    V2 = ho.G_KMS2_MPC_PER_MSUN * 1e14 / 1.0
    edges = np.quantile(x, np.linspace(0, 1, 11))
    for a, b in zip(edges[:-1], edges[1:]):
        sel = (x >= a) & (x < b)
        want = np.mean(V2 * ho.sigma_r2_over_v2(c * x[sel], np.array(c)))
        got = np.mean(v[sel] ** 2)
        m = 3 * sel.sum()
        assert abs(got / want - 1) < 5 * math.sqrt(2. / m) + 0.01


# ---- errors before any device work -----------------------------------------------------------------------------------------

def _halos(n=100, **kw):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ArrayCatalog, HaloCatalog
    rs = np.random.RandomState(1)
    cols = dict(Mass=10 ** rs.uniform(12, 14, n), Position=rs.uniform(0, 100, (n, 3)), Velocity=np.zeros((n, 3)))
    cols.update(kw)
    return HaloCatalog(ArrayCatalog(cols, comm=SelfComm(), BoxSize=100.), _cosmo(), 0.5)


def test_catalog_errors(monkeypatch):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ArrayCatalog, HaloCatalog, Zheng07Model
    from nbodykit_b200.source.catalog import halos as H

    def no_device(*a, **k):
        raise AssertionError("device work before the argument checks")
    monkeypatch.setattr(H._Halos, "run", no_device)
    src = ArrayCatalog(dict(Mass=np.ones(3), Position=np.zeros((3, 3)), Velocity=np.zeros((3, 3))), comm=SelfComm())
    with pytest.raises(ValueError, match="None"):
        HaloCatalog(src, _cosmo(), 0.5, mass=None)
    with pytest.raises(ValueError, match="missing"):
        HaloCatalog(src, _cosmo(), 0.5, velocity="Vel")
    with pytest.raises(TypeError):
        HaloCatalog({"Mass": 1}, _cosmo(), 0.5)
    with pytest.raises(NotImplementedError, match="halotools"):
        HaloCatalog(src, None, 0.5)
    with pytest.raises(ValueError):
        HaloCatalog(src, _cosmo(), 0.5, mdef="200q")
    halos = _halos()
    assert set(halos.columns) >= {"Mass", "Position", "Velocity", "VelocityOffset", "Concentration", "Radius"}
    assert halos.attrs["halo_mass_key"] == "halo_mvir" and halos.attrs["cosmo"] == _cosmo().pars
    halos["Concentration"] = np.full(100, 3.0)
    assert (np.asarray(halos["Concentration"].compute()) == 3.0).all()
    with pytest.raises(NotImplementedError, match="halotools"):
        halos.to_halotools()
    for bad in ("Zheng07Model", object(), 3):
        with pytest.raises(TypeError):
            halos.populate(bad, seed=1)
    with pytest.raises(ValueError, match="invalid"):
        halos.populate(Zheng07Model, seed=1, bad_param=2.)
    with pytest.raises(ValueError):
        halos.populate(Zheng07Model, seed=1, sigma_logM=0.)
    for seed in (-1, 1 << 32, 1.5, "3"):
        with pytest.raises(ValueError, match="seed"):
            halos.populate(Zheng07Model, seed=seed)
    for col in ("Mass", "Concentration"):
        for v in (0., -1., np.nan, np.inf):
            bad = _halos()
            arr = np.asarray(bad[col].compute(), dtype="f8").copy()
            arr[7] = v
            bad[col] = arr
            with pytest.raises(ValueError, match="non-finite or non-positive"):
                bad.populate(Zheng07Model, seed=1)
    nobox = HaloCatalog(ArrayCatalog(dict(Mass=np.ones(3) * 1e13, Position=np.zeros((3, 3)), Velocity=np.zeros((3, 3))),
                                     comm=SelfComm()), _cosmo(), 0.5)
    with pytest.raises(ValueError, match="BoxSize"):
        nobox.populate(Zheng07Model, seed=1)
    with pytest.raises(NotImplementedError, match="halotools"):
        Zheng07Model.to_halotools(_cosmo(), 0.5, "vir")


def test_models_and_exports():
    import nbodykit_b200.lab as lab
    from nbodykit_b200.hod import HODModel, Zheng07Model
    assert lab.HaloCatalog is not None and lab.Zheng07Model is Zheng07Model
    m = Zheng07Model()
    assert m.param_dict == DEFAULTS and m.modulate_with_cenocc
    assert issubclass(Zheng07Model, HODModel)
    with pytest.raises(ValueError):
        Zheng07Model(logMmax=3)


def test_to_halos_errors_without_running(monkeypatch):
    from nbodykit_b200.algorithms.fof import FOF
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ArrayCatalog
    monkeypatch.setattr(FOF, "run", lambda self: None)
    src = ArrayCatalog(dict(Position=np.random.RandomState(0).uniform(size=(10, 3))), comm=SelfComm(), BoxSize=1.)
    fof = FOF(src, 0.2, 5)
    for cosmo in (None, object()):
        with pytest.raises(NotImplementedError, match="halotools"):
            fof.to_halos(1e12, cosmo, 0.5)
    with pytest.raises(ValueError, match="posdef"):
        fof.to_halos(1e12, _cosmo(), 0.5, posdef="max")
    with pytest.raises(ValueError, match="Velocity"):
        fof.to_halos(1e12, _cosmo(), 0.5)
