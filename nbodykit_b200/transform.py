"""
Sky <-> Cartesian coordinate transforms (API of nbodykit/transform.py: SkyToUnitSphere, SkyToCartesian,
CartesianToEquatorial, CartesianToSky) and the halo relations (HaloRadius, HaloConcentration, HaloVelocityDispersion,
VectorProjection), in float64.

The reference works on dask arrays; here the inputs may be catalogue Columns, torch tensors (computed on their
device) or NumPy arrays, and the result is of the same kind: a Column if any input is one, else a tensor if any input
is one, else a NumPy array.  Only the ICRS frame is supported: other frames need astropy, which is not a dependency.

A `cosmo` may be any object with `comoving_distance(z)` (and, optionally, `efunc(z)`).  This package's Cosmology is
evaluated on the tensors where they are; any other cosmology is called on host float64 NumPy arrays, as the reference
calls it, and its result is moved back to the tensors' device.
"""
import math
import re

import numpy
import torch

from .base.catalog import Column, ConstantColumn
from .cosmology import C_KMS, Cosmology

__all__ = ['SkyToUnitSphere', 'SkyToCartesian', 'CartesianToEquatorial', 'CartesianToSky', 'HaloRadius', 'HaloConcentration',
           'HaloVelocityDispersion', 'VectorProjection']


def _check_frame(frame):
    if frame != 'icrs':
        raise NotImplementedError("frame '%s': only 'icrs' is supported (other frames need astropy)" % frame)


def _inputs(*args):
    """(the args as float64 tensors on one device, the wrap for the results)"""
    col = any(isinstance(a, Column) for a in args)
    vals = []
    for a in args:
        if isinstance(a, ConstantColumn):
            a = a.materialize()
        vals.append(a.compute() if isinstance(a, Column) else a)
    dev = next((v.device for v in vals if isinstance(v, torch.Tensor)), None)
    out = []
    for v in vals:
        t = v if isinstance(v, torch.Tensor) else torch.from_numpy(numpy.array(v, dtype='f8'))
        out.append(t.to(dtype=torch.float64, device=dev if dev is not None else t.device))
    if col:
        wrap = Column
    elif dev is not None:
        def wrap(t):
            return t
    else:
        def wrap(t):
            return t.cpu().numpy()
    return out, wrap


def _cosmo_call(fn, cosmo, z):
    """cosmo.<fn>(z) as a float64 tensor on z's device; only this package's Cosmology takes device tensors"""
    if isinstance(cosmo, Cosmology):
        v = getattr(cosmo, fn)(z)
    else:
        v = numpy.asarray(getattr(cosmo, fn)(z.detach().cpu().numpy()), dtype='f8')
    return torch.as_tensor(v, dtype=torch.float64, device=z.device).reshape(z.shape)


def _observer(observer, like):
    return torch.as_tensor(numpy.asarray(observer, dtype='f8').reshape(3), device=like.device)


def SkyToUnitSphere(ra, dec, degrees=True, frame='icrs'):
    """(N, 3) Cartesian unit vectors of (``ra``, ``dec``): (cos dec cos ra, cos dec sin ra, sin dec)"""
    _check_frame(frame)
    (ra, dec), wrap = _inputs(ra, dec)
    ra, dec = torch.broadcast_tensors(ra, dec)
    if degrees:
        ra, dec = torch.deg2rad(ra), torch.deg2rad(dec)
    cd = torch.cos(dec)
    return wrap(torch.stack([cd * torch.cos(ra), cd * torch.sin(ra), torch.sin(dec)], dim=-1))


def SkyToCartesian(ra, dec, redshift, cosmo, observer=[0, 0, 0], degrees=True, frame='icrs'):
    """(N, 3) Cartesian positions in Mpc/h: the unit vector of (``ra``, ``dec``) times ``cosmo.comoving_distance``
    of ``redshift``, plus ``observer``"""
    _check_frame(frame)
    (ra, dec, redshift), wrap = _inputs(ra, dec, redshift)
    ra, dec, redshift = torch.broadcast_tensors(ra, dec, redshift)
    pos = SkyToUnitSphere(ra, dec, degrees=degrees)
    r = _cosmo_call('comoving_distance', cosmo, redshift)
    return wrap(r[..., None] * pos + _observer(observer, pos))


def _equatorial(x, y, z):
    ra = torch.remainder(torch.rad2deg(torch.atan2(y, x)) - 360., 360.)
    dec = torch.rad2deg(torch.atan2(z, torch.hypot(x, y)))
    return ra, dec


def CartesianToEquatorial(pos, observer=[0, 0, 0], frame='icrs'):
    """(ra, dec) in degrees of the (N, 3) positions seen from ``observer``: RA in [0, 360), Dec in [-90, 90].  The
    result is stacked on the first axis, as the reference's, so ``ra, dec = CartesianToEquatorial(pos)`` works"""
    _check_frame(frame)
    (pos,), wrap = _inputs(pos)
    p = pos - _observer(observer, pos)
    ra, dec = _equatorial(p[..., 0], p[..., 1], p[..., 2])
    return wrap(torch.stack((ra, dec), dim=0))


def _redshift_of_distance(cosmo, r, zmax):
    """z with cosmo.comoving_distance(z) = r for 0 <= r <= comoving_distance(zmax): linear interpolation on the
    reference's grid (0 and 1024 log-spaced redshifts up to zmax), then Newton steps (slope c / H(z) when the cosmology
    has efunc, else that of the grid interval)"""
    zgrid = numpy.concatenate([[0.], numpy.logspace(-8, numpy.log10(zmax), 1024)])
    rgrid = numpy.asarray(cosmo.comoving_distance(zgrid), dtype='f8')
    if r.numel() and (not bool(torch.isfinite(r).all()) or float(r.max().item()) > rgrid[-1]):
        raise ValueError("CartesianToSky: a distance lies beyond comoving_distance(zmax = %g) = %g; raise zmax"
                         % (zmax, rgrid[-1]))
    zg = torch.from_numpy(zgrid).to(r.device)
    rg = torch.from_numpy(rgrid).to(r.device)
    k = torch.clamp(torch.searchsorted(rg, r, right=True) - 1, 0, len(zgrid) - 2)
    slope = (rg[k + 1] - rg[k]) / (zg[k + 1] - zg[k])
    z = zg[k] + (r - rg[k]) / slope
    for _ in range(8):
        d = _cosmo_call('comoving_distance', cosmo, z)
        if hasattr(cosmo, 'efunc'):
            slope = (C_KMS / 100.) / _cosmo_call('efunc', cosmo, z)
        z = z - (d - r) / slope
    return z


def CartesianToSky(pos, cosmo, velocity=None, observer=[0, 0, 0], zmax=100., frame='icrs'):
    r"""(ra, dec, z) of the (N, 3) positions in Mpc/h seen from ``observer``: RA and Dec in degrees, and the redshift
    whose comoving distance is the distance from the observer (``zmax`` bounds the search; a larger distance raises
    ValueError).  With ``velocity`` ((N, 3), km/s) the redshift-space redshift
    :math:`z + (v_\mathrm{pec} / c)(1 + z)` with :math:`v_\mathrm{pec} = \vec x \cdot \vec v / |\vec x|` is returned
    instead.  Stacked on the first axis, as the reference's"""
    _check_frame(frame)
    args = (pos,) if velocity is None else (pos, velocity)
    vals, wrap = _inputs(*args)
    p = vals[0] - _observer(observer, vals[0])
    ra, dec = _equatorial(p[..., 0], p[..., 1], p[..., 2])
    r = torch.linalg.vector_norm(p, dim=-1)
    z = _redshift_of_distance(cosmo, r, float(zmax))
    if velocity is not None:
        vpec = (p * vals[1]).sum(dim=-1) / r
        z = z + vpec / C_KMS * (1 + z)
    return wrap(torch.stack((ra, dec, z), dim=0))


# ---- halos ------------------------------------------------------------------------------------------------------------
def _halo_inputs(name, mass, cosmo, redshift):
    if not isinstance(cosmo, Cosmology):
        raise NotImplementedError("%s: only nbodykit_b200's Cosmology is supported (the reference hands other "
                                  "cosmologies to halotools and astropy, which are not dependencies)" % name)
    return _inputs(mass, redshift)


def _threshold(cosmo, z, mdef):
    """the density threshold of mdef at redshift z (tensor), in M_sun/h per (proper Mpc/h)^3"""
    rho = cosmo.rho_crit(z) * 1e10
    if mdef == 'vir':
        x = cosmo.Omega_m(z) - 1.
        return (18 * math.pi ** 2 + 82 * x - 39 * x * x) * rho
    m = re.fullmatch(r'(\d+)([cm])', mdef) if isinstance(mdef, str) else None
    if m is None or int(m.group(1)) <= 0:
        raise ValueError("mdef %r: expected 'vir', 'XXXc' or 'XXXm' with XXX a positive integer" % (mdef,))
    delta = float(m.group(1))
    return delta * rho if m.group(2) == 'c' else delta * cosmo.Omega_m(z) * rho


def HaloRadius(mass, cosmo, redshift, mdef='vir'):
    r"""the proper halo radius in Mpc/h of halos of ``mass`` (M_sun/h) for the mass definition ``mdef``:
    :math:`R = (3 M / (4 \pi \rho_\mathrm{thr}))^{1/3}` with :math:`\rho_\mathrm{thr} = \Delta \rho_c(z)` for
    ``'XXXc'``, :math:`\Delta \Omega_m(z) \rho_c(z)` for ``'XXXm'`` and :math:`\Delta_\mathrm{vir} \rho_c(z)` for
    ``'vir'``, with Bryan & Norman's (1998) :math:`\Delta_\mathrm{vir} = 18\pi^2 + 82x - 39x^2`,
    :math:`x = \Omega_m(z) - 1`.  Any other ``mdef`` raises ValueError"""
    (mass, redshift), wrap = _halo_inputs('HaloRadius', mass, cosmo, redshift)
    rho = _threshold(cosmo, redshift, mdef)
    return wrap((3 * mass / (4 * math.pi * rho)) ** (1. / 3))


def HaloConcentration(mass, cosmo, redshift, mdef='vir'):
    r"""the NFW concentration of halos of ``mass`` (M_sun/h): the virial fit of Dutton & Maccio (2014, eqs. 12-13),
    :math:`\log_{10} c = a + b \log_{10}(M / 10^{12} M_\odot/h)` with
    :math:`a = 0.537 + 0.488 e^{-0.718 z^{1.08}}` and :math:`b = -0.097 + 0.024 z`, for every ``mdef`` (which is
    still validated)"""
    (mass, redshift), wrap = _halo_inputs('HaloConcentration', mass, cosmo, redshift)
    _threshold(cosmo, redshift, mdef)
    a = 0.537 + (1.025 - 0.537) * torch.exp(-0.718 * redshift ** 1.08)
    b = -0.097 + 0.024 * redshift
    return wrap(10. ** (a + b * torch.log10(mass / 1e12)))


def HaloVelocityDispersion(mass, cosmo, redshift, mdef='vir'):
    r"""the velocity dispersion in km/s of halos of ``mass`` (M_sun/h), the reference's model (Evrard et al. 2008):
    :math:`1100 (E(z) M / 10^{15})^{0.33333}`"""
    (mass, redshift), wrap = _halo_inputs('HaloVelocityDispersion', mass, cosmo, redshift)
    return wrap(1100. * (cosmo.efunc(redshift) * mass / 1e15) ** 0.33333)


def VectorProjection(vector, direction):
    r"""the components of the (..., D) ``vector`` along ``direction`` (D,):
    :math:`(\mathbf{v} \cdot \hat{\mathbf{d}}) \hat{\mathbf{d}}` with :math:`\hat{\mathbf{d}} = \mathbf{d} / |\mathbf{d}|`
    (``direction`` need not be normalised)"""
    (vector,), wrap = _inputs(vector)
    d = torch.as_tensor(numpy.asarray(direction, dtype='f8'), device=vector.device)
    d = d / (d ** 2).sum() ** 0.5
    proj = (vector * d).sum(dim=-1)
    return wrap(proj[..., None] * d)
