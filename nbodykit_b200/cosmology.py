"""
Self-contained stand-ins for the two things this package needs from `nbodykit.cosmology` (the reference gets both from
CLASS via classylss, which is not part of this package -- SURVEY.md §2.1):

`NoWiggleEHPower` is the Eisenstein & Hu (1998) zero-baryon-oscillation fitting formula (their
eqs. 26, 28-31), normalised to sigma8 with a top-hat window; the same shape the reference offers as
`LinearPower(cosmo, z, transfer='NoWiggleEisensteinHu')` (cosmology/power/transfers.py:184-255).

`Cosmology` is a background-only LambdaCDM model (E(z), the comoving distance) for the sky <-> Cartesian transforms
of transform.py; `Planck15` is an instance of it.
"""
import math

import numpy


class NoWiggleEHPower(object):
    def __init__(self, h=0.6774, Omega0_m=0.3089, Omega0_b=0.0486, n_s=0.9667, sigma8=0.8159, Tcmb=2.7255,
                 redshift=0.0, growth=1.0):
        self.h, self.Om, self.Ob, self.n_s, self.sigma8 = h, Omega0_m, Omega0_b, n_s, sigma8
        self.redshift = redshift
        self.growth = growth          # D(z)/D(0), supplied by the caller (no background solver here)
        self.theta = Tcmb / 2.7
        omh2 = self.Om * h * h
        obh2 = self.Ob * h * h
        fb = self.Ob / self.Om
        # sound horizon (EH98 eq. 26) and alpha_gamma (eq. 31)
        self.s = 44.5 * numpy.log(9.83 / omh2) / numpy.sqrt(1 + 10 * obh2 ** 0.75)
        self.alpha = 1 - 0.328 * numpy.log(431 * omh2) * fb + 0.38 * numpy.log(22.3 * omh2) * fb * fb
        self._norm = 1.0
        self._norm = (sigma8 / self.sigma_r(8.0)) ** 2

    def transfer(self, k):
        """k in h/Mpc"""
        k = numpy.asarray(k, dtype='f8')
        kmpc = k * self.h                       # 1/Mpc
        omh2 = self.Om * self.h ** 2
        gamma_eff = omh2 * (self.alpha + (1 - self.alpha) / (1 + (0.43 * kmpc * self.s) ** 4))   # eq. 30
        q = kmpc * self.theta ** 2 / gamma_eff                                                       # eq. 28
        L0 = numpy.log(2 * numpy.e + 1.8 * q)
        C0 = 14.2 + 731.0 / (1 + 62.5 * q)
        return L0 / (L0 + C0 * q * q)                                                                 # eq. 29

    def __call__(self, k):
        k = numpy.asarray(k, dtype='f8')
        with numpy.errstate(invalid='ignore', divide='ignore'):
            p = self._norm * self.growth ** 2 * k ** self.n_s * self.transfer(k) ** 2
        return numpy.where(k > 0, p, 0.0)

    def sigma_r(self, r, kmin=1e-5, kmax=1e2, n=4096):
        """rms of the top-hat smoothed linear field at radius r [Mpc/h]"""
        lnk = numpy.linspace(numpy.log(kmin), numpy.log(kmax), n)
        k = numpy.exp(lnk)
        x = k * r
        w = 3 * (numpy.sin(x) - x * numpy.cos(x)) / x ** 3
        integrand = k ** 3 * self(k) * w * w / (2 * numpy.pi ** 2)
        return numpy.sqrt(numpy.trapezoid(integrand, lnk))


LinearPower = NoWiggleEHPower


# ---- background ------------------------------------------------------------------------------------------------------
C_KMS = 299792.458                      # speed of light [km/s]
# Omega_gamma h^2 per K^4: a_rad T^4 8 pi G / (3 c^2 (100 km/s/Mpc)^2), a_rad = 4 sigma_SB / c (CODATA 2018, SI)
_SIGMA_SB, _C_SI, _G_SI, _MPC_M = 5.670374419e-8, 299792458.0, 6.67430e-11, 3.0856775814913673e22
_OMEGA_G_H2_PER_K4 = (4 * _SIGMA_SB / _C_SI) * 8 * math.pi * _G_SI / (3 * _C_SI ** 2 * (1e5 / _MPC_M) ** 2)
# the solar mass: the IAU 2015 nominal GM_sun (resolution B3) over G, in kg
_GM_SUN_SI = 1.3271244e20
M_SUN_KG = _GM_SUN_SI / _G_SI
# G in (km/s)^2 Mpc / M_sun, and the critical density today in 10^10 (M_sun/h) / (Mpc/h)^3 (CLASS's unit for rho_crit)
G_KMS2_MPC_PER_MSUN = _GM_SUN_SI / _MPC_M / 1e6
RHO_CRIT0 = 3 * 100. ** 2 / (8 * math.pi * G_KMS2_MPC_PER_MSUN) / 1e10
_DU = 1. / 64                           # table nodes: uniform in ln(1 + z)
_GL_X, _GL_W = numpy.polynomial.legendre.leggauss(8)


class Cosmology(object):
    r"""
    A background-only cosmology: LambdaCDM with photons (temperature ``T0_cmb``) and ``N_ur`` massless neutrino
    species as radiation, baryons and cold dark matter as matter, curvature ``Omega0_k``, and a cosmological constant
    closing the budget.  Only the expansion history is modelled:

    .. math::

        E(z) = \sqrt{\Omega_r (1+z)^4 + \Omega_m (1+z)^3 + \Omega_k (1+z)^2 + \Omega_\Lambda}

    with :math:`\Omega_r = \Omega_\gamma (1 + \tfrac{7}{8} (4/11)^{4/3} N_{ur})` and
    :math:`\Omega_\Lambda = 1 - \Omega_m - \Omega_r - \Omega_k`.  Parameter names follow the reference's
    (CLASS) names; there are no massive neutrinos, perturbations or dark-energy fluids.

    Every algorithm that takes a ``cosmo`` needs only its ``comoving_distance(z)``, so any object with that method
    may be passed instead.
    """

    def __init__(self, h=0.67556, T0_cmb=2.7255, Omega0_b=0.022032 / 0.67556 ** 2, Omega0_cdm=0.12038 / 0.67556 ** 2,
                 N_ur=3.046, Omega0_k=0.):
        pars = dict(h=h, T0_cmb=T0_cmb, Omega0_b=Omega0_b, Omega0_cdm=Omega0_cdm, N_ur=N_ur, Omega0_k=Omega0_k)
        for k, v in pars.items():
            if not numpy.isfinite(v):
                raise ValueError("Cosmology: %s must be finite (got %r)" % (k, v))
        if h <= 0 or T0_cmb < 0 or N_ur < 0:
            raise ValueError("Cosmology: h must be positive, T0_cmb and N_ur non-negative")
        self.pars = {k: float(v) for k, v in pars.items()}
        for k, v in self.pars.items():
            setattr(self, k, v)
        self.Omega0_g = _OMEGA_G_H2_PER_K4 * T0_cmb ** 4 / h ** 2
        self.Omega0_ur = N_ur * 7. / 8. * (4. / 11.) ** (4. / 3.) * self.Omega0_g
        self.Omega0_r = self.Omega0_g + self.Omega0_ur
        self.Omega0_m = Omega0_b + Omega0_cdm
        self.Omega0_lambda = 1. - self.Omega0_m - self.Omega0_r - Omega0_k
        self._tables = {}

    @classmethod
    def from_dict(cls, pars):
        """the cosmology of a :attr:`pars` dictionary"""
        return cls(**pars)

    def __repr__(self):
        return "Cosmology(%s)" % ", ".join("%s=%r" % kv for kv in self.pars.items())

    def __eq__(self, other):
        return isinstance(other, Cosmology) and self.pars == other.pars

    def __hash__(self):
        return hash(tuple(sorted(self.pars.items())))

    def efunc(self, z):
        """E(z) = H(z) / H0; NumPy arrays / scalars, or torch tensors (computed where they are)"""
        sqrt = _backend(z)[1]
        a1 = 1. + z
        return sqrt(((self.Omega0_r * a1 + self.Omega0_m) * a1 + self.Omega0_k) * a1 * a1 + self.Omega0_lambda)

    def Omega_m(self, z):
        r"""the matter density parameter at redshift z, :math:`\Omega_m (1+z)^3 / E(z)^2`; NumPy arrays / scalars, or
        torch tensors (computed where they are)"""
        a1 = 1. + z
        return self.Omega0_m * a1 * a1 * a1 / self.efunc(z) ** 2

    def rho_crit(self, z):
        r"""the critical density :math:`3 H(z)^2 / (8 \pi G)` in :math:`10^{10} (M_\odot/h) / (\mathrm{Mpc}/h)^3`
        (CLASS's name and unit); NumPy arrays / scalars, or torch tensors (computed where they are)"""
        return RHO_CRIT0 * self.efunc(z) ** 2

    def _integral(self, z0, z1):
        """(c / 100) int_{z0}^{z1} dz / E(z) in Mpc/h, 8-point Gauss-Legendre, elementwise"""
        mid, half = 0.5 * (z0 + z1), 0.5 * (z1 - z0)
        acc = 0.
        for x, w in zip(_GL_X, _GL_W):
            acc = acc + float(w) / self.efunc(mid + float(x) * half)
        return (C_KMS / 100.) * half * acc

    def _table(self, umax, like):
        """(z nodes, comoving distance at the nodes) covering ln(1 + z) <= umax, on the device of `like`"""
        import torch
        key = (str(like.device) if isinstance(like, torch.Tensor) else 'numpy')
        t = self._tables.get(key)
        if t is None or t[0] < umax:
            k = int(math.ceil(max(umax, 1.) / _DU)) + 1
            z = numpy.expm1(numpy.arange(k + 1) * _DU)
            chi = numpy.concatenate([[0.], numpy.cumsum(self._integral(z[:-1], z[1:]))])
            zt, ct = (torch.from_numpy(z).to(like.device), torch.from_numpy(chi).to(like.device)) \
                if key != 'numpy' else (z, chi)
            t = self._tables[key] = (k * _DU, zt, ct)
        return t[1], t[2]

    def comoving_distance(self, z):
        r"""the line-of-sight comoving distance :math:`\frac{c}{H_0} \int_0^z dz' / E(z')` in Mpc/h, for z > -1.
        NumPy arrays / scalars (float64 result), or torch tensors (float64, on their device).  The distance to the
        ln(1 + z) node below z comes from a table built once by Gauss-Legendre quadrature over nodes 1/64 apart; the
        rest is one more Gauss-Legendre integral, so the result is accurate to a few units of double rounding."""
        import torch
        is_t = isinstance(z, torch.Tensor)
        if is_t:
            zz = z.to(torch.float64)
        else:
            zz = numpy.asarray(z, dtype='f8')
        if zz.numel() if is_t else zz.size:
            zmax = float(zz.max().item()) if is_t else float(zz.max())
            if not numpy.isfinite(zmax) or (float(zz.min().item()) if is_t else float(zz.min())) <= -1:
                raise ValueError("comoving_distance: redshifts must be finite and above -1")
        else:
            zmax = 0.
        znode, chi = self._table(math.log1p(max(zmax, 0.)), zz)
        u = torch.log1p(zz) if is_t else numpy.log1p(zz)
        if is_t:
            k = torch.clamp(torch.floor(u / _DU), 0, znode.numel() - 2).to(torch.int64)
        else:
            k = numpy.clip(numpy.floor(u / _DU), 0, len(znode) - 2).astype('i8')
        out = chi[k] + self._integral(znode[k], zz)
        return out if is_t or out.ndim else float(out)


def _backend(x):
    import torch
    if isinstance(x, torch.Tensor):
        return torch, torch.sqrt
    return numpy, numpy.sqrt


# Planck 2015 (astropy's Planck15: H0 = 67.74, Om0 = 0.3075, Ob0 = 0.0486, Tcmb0 = 2.7255 K, Neff = 3.046 with one
# 0.06 eV neutrino), as the reference builds it for CLASS (N_ur = 2.0328).  This is not CLASS's Planck15: the massive
# neutrino is counted here as matter at all redshifts (Omega_nu h^2 = 0.06 / 93.14), and how far the distances are
# from CLASS's has not been checked.
Planck15 = Cosmology(h=0.6774, T0_cmb=2.7255, Omega0_b=0.0486,
                     Omega0_cdm=0.3075 - 0.0486 + 0.06 / 93.14 / 0.6774 ** 2, N_ur=2.0328, Omega0_k=0.)
