"""CPU checks of the survey layer: the background cosmology's comoving distance against quadrature and closed forms,
the sky <-> Cartesian transforms, the '__cosmo__' JSON round trip, the argument errors of SurveyDataPairCount /
SurveyData2PCF / SurveyData3PCF, and oracle/survey_paircount_oracle.py against its own brute force."""
import json

import numpy as np
import pytest
import torch

from oracle import survey_paircount_oracle as so

C_H0 = 299792.458 / 100.


def test_comoving_distance_against_quad():
    from scipy.integrate import quad
    from nbodykit_b200.cosmology import Cosmology, Planck15
    z = np.array([0., 1e-6, 1e-3, 0.05, 0.3, 0.5, 1., 2.5, 7., 30., 100., 1100.])
    for c in (Planck15, Cosmology(), Cosmology(h=0.7, Omega0_b=0.04, Omega0_cdm=0.2, Omega0_k=0.05, N_ur=2.)):
        want = np.array([quad(lambda x: C_H0 / c.efunc(x), 0., zz, epsabs=0., epsrel=1e-13, limit=500)[0] for zz in z])
        got = c.comoving_distance(z)
        assert got.dtype == np.float64 and got.shape == z.shape
        np.testing.assert_allclose(got, want, rtol=1e-9, atol=0)
        # scalars, unsorted input and torch tensors give the same values
        assert c.comoving_distance(0.5) == got[5]
        p = np.random.RandomState(0).permutation(len(z))
        np.testing.assert_array_equal(c.comoving_distance(z[p]), got[p])
        t = c.comoving_distance(torch.from_numpy(z))
        assert isinstance(t, torch.Tensor) and t.dtype == torch.float64
        np.testing.assert_allclose(t.numpy(), got, rtol=1e-15, atol=0)


def test_comoving_distance_closed_forms():
    from nbodykit_b200.cosmology import Cosmology
    z = np.concatenate([[0.], np.logspace(-7, 3, 60)])
    # Einstein-de Sitter: chi = 2 c / H0 (1 - 1 / sqrt(1 + z)), written without cancellation at small z
    eds = Cosmology(h=0.7, T0_cmb=0., N_ur=0., Omega0_b=0.05, Omega0_cdm=0.95)
    assert eds.Omega0_r == 0. and abs(eds.Omega0_lambda) < 1e-15
    q = np.sqrt(1. + z)
    np.testing.assert_allclose(eds.comoving_distance(z), 2. * C_H0 * z / (q * (1. + q)), rtol=1e-12, atol=0)
    # pure Lambda: E = 1, chi = c z / H0
    lam = Cosmology(h=0.7, T0_cmb=0., N_ur=0., Omega0_b=0., Omega0_cdm=0.)
    np.testing.assert_allclose(lam.comoving_distance(z), C_H0 * z, rtol=1e-12, atol=0)


def test_cosmology_pars_and_errors():
    from nbodykit_b200.cosmology import Cosmology, Planck15
    c = Cosmology.from_dict(Planck15.pars)
    assert c == Planck15 and c.pars == Planck15.pars
    assert abs(Planck15.Omega0_m + Planck15.Omega0_r + Planck15.Omega0_lambda - 1.) < 1e-15
    with pytest.raises(ValueError):
        Cosmology(h=-1.)
    with pytest.raises(ValueError):
        Cosmology(Omega0_k=np.nan)
    with pytest.raises(ValueError):
        Planck15.comoving_distance([0.1, -1.])


def test_foreign_cosmology_gets_host_arrays():
    """a cosmology with only comoving_distance, written for NumPy, works from tensors and from arrays"""
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200 import transform as T

    class TableCosmo(object):
        def __init__(self):
            self.z = np.linspace(0., 3., 30001)
            self.d = Planck15.comoving_distance(self.z)

        def comoving_distance(self, z):
            assert isinstance(z, np.ndarray) and z.dtype == np.float64
            return np.interp(z, self.z, self.d)
    c = TableCosmo()
    rng = np.random.RandomState(3)
    pos = rng.normal(size=(500, 3)) * 800.
    for p in (pos, torch.from_numpy(pos)):
        ra, dec, z = T.CartesianToSky(p, c)
        back = T.SkyToCartesian(ra, dec, z, c)
        assert type(back) is type(p)
        np.testing.assert_allclose(np.asarray(back), pos, rtol=0, atol=1e-9)
    # the table interpolates Planck15 closely
    np.testing.assert_allclose(z.numpy(), T.CartesianToSky(pos, Planck15)[2], rtol=1e-7)


def test_sky_cartesian_round_trip():
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200 import transform as T
    from nbodykit_b200.base.catalog import Column
    rng = np.random.RandomState(1)
    pos = rng.normal(size=(2000, 3)) * 800.
    obs = [10., -20., 5.]
    ra, dec, z = T.CartesianToSky(pos, Planck15, observer=obs)
    assert ra.min() >= 0 and ra.max() < 360 and np.abs(dec).max() <= 90
    back = T.SkyToCartesian(ra, dec, z, Planck15, observer=obs)
    np.testing.assert_allclose(back, pos, rtol=0, atol=1e-9)
    # tensors in, tensors out; Columns in, Columns out
    rt, dt, zt = T.CartesianToSky(torch.from_numpy(pos), Planck15, observer=obs)
    np.testing.assert_allclose(zt.numpy(), z, rtol=1e-14)
    c = T.SkyToCartesian(Column(ra), Column(dec), Column(z), Planck15, observer=obs)
    assert isinstance(c, Column)
    np.testing.assert_array_equal(np.asarray(c), back)
    u = T.SkyToUnitSphere(ra, dec)
    np.testing.assert_allclose(np.linalg.norm(u, axis=1), 1., rtol=1e-15)
    # velocities: z + (v . x / |x| / c) (1 + z)
    v = rng.normal(size=pos.shape) * 300.
    zv = T.CartesianToSky(pos, Planck15, velocity=v, observer=obs)[2]
    x = pos - obs
    vpec = (x * v).sum(-1) / np.linalg.norm(x, axis=-1)
    np.testing.assert_allclose(zv, z + vpec / 299792.458 * (1 + z), rtol=1e-14)
    with pytest.raises(ValueError):
        T.CartesianToSky(np.array([[1e5, 0., 0.]]), Planck15, zmax=2.)
    with pytest.raises(NotImplementedError):
        T.SkyToCartesian(ra, dec, z, Planck15, frame='galactic')


def test_cartesian_to_equatorial_against_numpy():
    from nbodykit_b200 import transform as T
    rng = np.random.RandomState(2)
    pos = rng.normal(size=(1000, 3))
    pos[:4] = [[1., 0., 0.], [-1., 0., 0.], [0., -1., 0.], [0., 0., 1.]]
    ra, dec = T.CartesianToEquatorial(pos, observer=[0.5, 0., 0.])
    x, y, z = (pos - [0.5, 0., 0.]).T
    want_ra = np.mod(np.rad2deg(np.arctan2(y, x)) - 360., 360.)
    want_dec = np.rad2deg(np.arctan2(z, np.hypot(x, y)))
    np.testing.assert_allclose(ra, want_ra, rtol=1e-15, atol=1e-13)
    np.testing.assert_allclose(dec, want_dec, rtol=1e-15, atol=1e-13)
    r0, d0 = T.CartesianToEquatorial(pos[:4])
    assert r0[0] == 0. and r0[1] == 180. and r0[2] == 270. and d0[3] == 90.


def test_cosmo_json_round_trip(tmp_path):
    from nbodykit_b200.cosmology import Cosmology, Planck15
    from nbodykit_b200.utils import JSONDecoder, JSONEncoder
    c = Cosmology(h=0.7, Omega0_k=0.01)
    s = json.dumps({'attrs': {'cosmo': c, 'other': Planck15, 'edges': np.arange(3.)}}, cls=JSONEncoder)
    assert '"__cosmo__"' in s
    d = json.loads(s, cls=JSONDecoder)
    assert d['attrs']['cosmo'] == c and d['attrs']['other'] == Planck15
    # other values encode as before
    assert json.dumps({'a': np.arange(2)}, cls=JSONEncoder) == \
        '{"a": {"__dtype__": "<i8", "__shape__": [2], "__data__": [0, 1]}}'


_COMM = []


def _sky_cat(cols):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ArrayCatalog
    if not _COMM:
        _COMM.append(SelfComm())
    return ArrayCatalog({k: np.asarray(v) for k, v in cols.items()}, comm=_COMM[0])


def test_argument_errors():
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200.lab import SurveyData2PCF, SurveyData3PCF, SurveyDataPairCount
    ra, dec, z = so.sky_catalogue(0, 10)
    full = _sky_cat(dict(RA=ra, DEC=dec, Redshift=z))
    nored = _sky_cat(dict(RA=ra, DEC=dec))
    edges = np.linspace(1., 10., 4)
    with pytest.raises(ValueError, match="Redshift"):
        SurveyDataPairCount('1d', nored, edges, cosmo=Planck15)
    with pytest.raises(ValueError, match="DEC"):
        SurveyDataPairCount('angular', _sky_cat(dict(RA=ra)), edges)
    with pytest.raises(ValueError, match="missing"):
        SurveyDataPairCount('1d', full, edges, cosmo=Planck15, second=nored)
    with pytest.raises(ValueError, match="cosmo"):
        SurveyDataPairCount('2d', full, edges, Nmu=5)
    with pytest.raises(ValueError, match="lower edge"):
        SurveyDataPairCount('angular', nored, [0., 1., 2.])
    with pytest.raises(ValueError, match="180"):
        SurveyDataPairCount('angular', nored, [1., 90., 180.5])
    with pytest.raises(ValueError, match="Nmu"):
        SurveyDataPairCount('2d', full, edges, cosmo=Planck15)
    with pytest.raises(ValueError, match="'2d'"):
        SurveyDataPairCount('1d', full, edges, cosmo=Planck15, Nmu=4)
    with pytest.raises(ValueError, match="pimax"):
        SurveyDataPairCount('projected', full, edges, cosmo=Planck15)
    with pytest.raises(ValueError, match="projected"):
        SurveyDataPairCount('2d', full, edges, cosmo=Planck15, Nmu=3, pimax=10.)
    with pytest.raises(ValueError, match="at least 1.0"):
        SurveyDataPairCount('projected', full, edges, cosmo=Planck15, pimax=0.5)
    with pytest.raises(ValueError, match="allowed"):
        SurveyDataPairCount('3d', full, edges, cosmo=Planck15)
    with pytest.raises(ValueError, match="strictly increasing"):
        SurveyDataPairCount('1d', full, [3., 2., 4.], cosmo=Planck15)
    with pytest.raises(ValueError, match="cosmo"):
        SurveyData2PCF('1d', full, full, edges)
    with pytest.raises(ValueError, match="Redshift"):
        SurveyData3PCF(nored, [0, 1], edges, Planck15)
    with pytest.raises(ValueError, match="poles"):
        SurveyData3PCF(full, [0, 0], edges, Planck15)


@pytest.mark.parametrize("mode", ["1d", "2d", "projected", "angular"])
def test_oracle_against_brute_force(mode):
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200 import transform as T
    ra, dec, z = so.sky_catalogue(3, 500, ra=(150., 170.), dec=(0., 15.), z=(0.1, 0.01))
    if mode == "angular":
        pos = T.SkyToUnitSphere(ra, dec)
        edges, kw = np.logspace(-1, 1.2, 7), {}
    else:
        pos = T.SkyToCartesian(ra, dec, z, Planck15)
        edges = np.linspace(2., 40., 8)
        kw = dict(Nmu=5) if mode == "2d" else dict(pimax=20.) if mode == "projected" else {}
    # a pair along one line of sight (mu = 1), a pair through the observer (l = 0) and a pair on an edge
    pos = np.concatenate([pos, [pos[0] * 1.03, -pos[1], pos[2] * (1 + edges[2] / np.linalg.norm(pos[2]))]])
    w = np.random.RandomState(4).uniform(0.5, 2., len(pos))
    cross = np.random.RandomState(5).permutation(pos)[:300]
    for p2, w1 in ((None, w), (cross, None)):
        a = so.count(pos, mode, edges, pos2=p2, w1=w1, **kw)
        b = so.brute_force(pos, mode, edges, pos2=p2, w1=w1, **kw)
        np.testing.assert_array_equal(a["npairs"], b["npairs"])
        np.testing.assert_allclose(a["wnpairs"], b["wnpairs"], rtol=1e-13)
        np.testing.assert_allclose(a["sepsum"], b["sepsum"], rtol=1e-13)
        assert a["npairs"].sum() > 500
    if mode == "2d":
        assert b["npairs"][:, -1].sum() > 0
