"""
Halo occupation models (API of nbodykit/hod.py: HODModel, Zheng07Model, Leauthaud11Model, Hearin15Model) for
:meth:`HaloCatalog.populate`.

The reference converts these classes to halotools models and lets halotools populate the halos on the CPU.  Here the
models are evaluated by this package's own kernels (csrc/hod.cu) to the contract of DESIGN.md 4.13; halotools is not a
dependency, so :meth:`HODModel.to_halotools` raises NotImplementedError.

The stellar-to-halo-mass relation
---------------------------------
Leauthaud11Model and Hearin15Model need the mean log stellar mass of a halo of mass M, the inverse of the Behroozi et
al. (2010) relation M_h(M*).  As halotools does, :func:`smhm_spline` tabulates log10 M_h at 100 values of log10 M* on
[8.5, 12.5] and fits scipy's cubic ``InterpolatedUnivariateSpline`` to (log10 M_h, log10 M*); the kernel evaluates its
knots and coefficients as FITPACK's ``splev`` does, extrapolating outside the table.

The Jeans table
---------------
The radial velocity dispersion of a satellite at y = r / r_s in an NFW halo of concentration c is (isotropic Jeans
equation, Lokas & Mamon 2001)

    sigma_r^2 = V^2 c / g(c) y (1 + y)^2 I(y),    I(y) = int_y^inf g(t) / (t^3 (1 + t)^2) dt,

with g(y) = ln(1 + y) - y / (1 + y) and V^2 = G M / R.  I(y) does not depend on c, so it is tabulated once on the host:
ln I and its derivative in s = ln y at nodes 1/128 apart over s in [-20, 24], from 8-point Gauss-Legendre panels
between nodes summed from the top, the tail above the top integrated the same way out to s = 64.  The kernel
interpolates ln I by cubic Hermite polynomials; outside the table it uses the leading terms of the series at 0 and at
infinity.
"""
import math

import numpy

__all__ = ['HODModel', 'Zheng07Model', 'Leauthaud11Model', 'Hearin15Model']


class HODModel(object):
    """
    A halo occupation model: a set of named parameters (:attr:`param_dict`) that :meth:`HaloCatalog.populate` reads.
    Pass the class (its default parameters) or an instance.
    """
    defaults = {}

    def __init__(self, **params):
        self.param_dict = dict(self.defaults)
        self.update(params)

    def update(self, params):
        """set parameters; an unknown name raises ValueError"""
        missing = set(params) - set(self.defaults)
        if missing:
            raise ValueError("invalid halo model parameter names: %s" % str(sorted(missing)))
        self.param_dict.update({k: float(v) for k, v in params.items()})

    @staticmethod
    def to_halotools(cosmo, redshift, mdef, concentration_key=None, **kwargs):
        """the halotools model of the reference; halotools is not a dependency of this package"""
        raise NotImplementedError("HODModel.to_halotools needs halotools, which is not a dependency of nbodykit_b200; "
                                  "HaloCatalog.populate evaluates the model on the GPU instead")


class Zheng07Model(HODModel):
    r"""
    The HOD of Zheng et al. (2007), with halotools' parameter names and its luminosity-threshold -20 defaults.

    - centrals: :math:`\langle N_\mathrm{cen} \rangle = \frac{1}{2}[1 + \mathrm{erf}((\log_{10} M - \log M_\mathrm{min})
      / \sigma_{\log M})]`
    - satellites: :math:`\langle N_\mathrm{sat} \rangle = ((M - M_0) / M_1)^\alpha` above :math:`M_0`, times
      :math:`\langle N_\mathrm{cen} \rangle` when ``modulate_with_cenocc`` (the reference's default)

    Parameters
    ----------
    modulate_with_cenocc : bool, optional
        multiply the satellite mean by the central occupation
    **params :
        ``logMmin``, ``sigma_logM``, ``logM0``, ``logM1``, ``alpha``
    """
    defaults = dict(logMmin=12.02, sigma_logM=0.26, logM0=11.38, logM1=13.31, alpha=1.06)
    gal_types = ('centrals', 'satellites')

    def __init__(self, modulate_with_cenocc=True, **params):
        self.modulate_with_cenocc = bool(modulate_with_cenocc)
        HODModel.__init__(self, **params)

    def arguments(self):
        """the constructor arguments other than the parameters"""
        return dict(modulate_with_cenocc=self.modulate_with_cenocc)

    @staticmethod
    def to_halotools(cosmo, redshift, mdef, concentration_key=None, **kwargs):
        """the halotools model of the reference; halotools is not a dependency of this package"""
        raise NotImplementedError("Zheng07Model.to_halotools needs halotools, which is not a dependency of "
                                  "nbodykit_b200; HaloCatalog.populate evaluates the model on the GPU instead")

    def check(self):
        """ValueError unless every parameter is finite and sigma_logM positive"""
        p = self.param_dict
        for k, v in p.items():
            if not math.isfinite(v):
                raise ValueError("Zheng07Model: %s must be finite (got %r)" % (k, v))
        if not p['sigma_logM'] > 0:
            raise ValueError("Zheng07Model: sigma_logM must be positive (got %r)" % p['sigma_logM'])
        if not (math.isfinite(10. ** p['logM0']) and 0 < 10. ** p['logM1'] < math.inf):
            raise ValueError("Zheng07Model: 10^logM0 and 10^logM1 must be finite and 10^logM1 positive")


# ---- the stellar-to-halo-mass relation ------------------------------------------------------------------------------
SMHM_LITTLE_H = 0.7                                  # the h of Behroozi et al. (2010)
SMHM_LOGMS = numpy.linspace(8.5, 12.5, 100)          # log10 M* (Msun/h^2) of the table that is inverted
SMHM_DEFAULTS = dict(smhm_m0_0=10.72, smhm_m0_a=0.59, smhm_m1_0=12.35, smhm_m1_a=0.3, smhm_beta_0=0.43,
                     smhm_beta_a=0.18, smhm_delta_0=0.56, smhm_delta_a=0.18, smhm_gamma_0=1.54, smhm_gamma_a=2.52,
                     scatter_model_param1=0.2)


def behroozi10_log_mhalo(logms, params, redshift):
    r"""log10 of the halo mass (Msun/h) of mean stellar mass 10^logms (Msun/h^2), Behroozi et al. (2010) at `redshift`:
    with a = 1 / (1 + z), X(a) = X_0 + X_a (a - 1) and r = M* h^2 / 10^m0,
    :math:`\log_{10} M_h = m_1 + \beta \log_{10} r + r^\delta / (1 + r^{-\gamma}) - 1/2` in Msun, times h"""
    a = 1.0 / (1.0 + float(redshift))
    p = params
    m0 = p['smhm_m0_0'] + p['smhm_m0_a'] * (a - 1.0)
    m1 = p['smhm_m1_0'] + p['smhm_m1_a'] * (a - 1.0)
    beta = p['smhm_beta_0'] + p['smhm_beta_a'] * (a - 1.0)
    delta = p['smhm_delta_0'] + p['smhm_delta_a'] * (a - 1.0)
    gamma = p['smhm_gamma_0'] + p['smhm_gamma_a'] * (a - 1.0)
    r = 10.0 ** numpy.asarray(logms, dtype='f8') * SMHM_LITTLE_H ** 2 / 10.0 ** m0
    with numpy.errstate(over='ignore', divide='ignore', invalid='ignore'):
        lmh = m1 + beta * numpy.log10(r) + r ** delta / (1.0 + r ** (-gamma)) - 0.5
    return lmh + numpy.log10(SMHM_LITTLE_H)


def smhm_spline(params, redshift):
    """(t, c): the knots and coefficients of the cubic spline log10 M_h -> mean log10 M* (scipy's
    InterpolatedUnivariateSpline through the inverted Behroozi table); ValueError unless the table is finite and
    increasing"""
    from scipy.interpolate import InterpolatedUnivariateSpline
    lmh = behroozi10_log_mhalo(SMHM_LOGMS, params, redshift)
    if not (numpy.isfinite(lmh).all() and (numpy.diff(lmh) > 0).all()):
        raise ValueError("the Behroozi10 stellar-to-halo-mass relation of these parameters is not finite and "
                         "increasing over log10 M* in [8.5, 12.5] at redshift %r" % float(redshift))
    t, c, k = InterpolatedUnivariateSpline(lmh, SMHM_LOGMS, k=3)._eval_args
    assert k == 3
    return numpy.ascontiguousarray(t, 'f8'), numpy.ascontiguousarray(c, 'f8')


class Leauthaud11Model(HODModel):
    r"""
    The stellar-mass-threshold HOD of Leauthaud et al. (2011), with halotools' parameter names and defaults, on the
    Behroozi et al. (2010) stellar-to-halo-mass relation (DESIGN.md 4.13).

    - centrals: :math:`\langle N_\mathrm{cen} \rangle = \frac{1}{2}[1 - \mathrm{erf}((t - \log_{10} M_*(M)) /
      (\sqrt{2}\,\sigma))]`, with :math:`M_*(M)` the inverted relation and :math:`\sigma` = ``scatter_model_param1``
    - satellites: :math:`\langle N_\mathrm{sat} \rangle = (M / M_\mathrm{sat})^{\alpha_\mathrm{sat}}
      \exp(-M_\mathrm{cut} / M)`, :math:`M_\mathrm{sat} = 10^{12} b_\mathrm{sat} (M_\mathrm{knee} / 10^{12})^{\beta_
      \mathrm{sat}}`, :math:`M_\mathrm{cut} = 10^{12} b_\mathrm{cut} (M_\mathrm{knee} / 10^{12})^{\beta_\mathrm{cut}}`
      with :math:`M_\mathrm{knee} = M_h(t)`, times :math:`\langle N_\mathrm{cen} \rangle` when ``modulate_with_cenocc``

    Parameters
    ----------
    threshold : float, optional
        the stellar-mass threshold t, log10 M* in Msun/h^2
    modulate_with_cenocc : bool, optional
        multiply the satellite mean by the central occupation
    **params :
        the ``smhm_*`` parameters, ``scatter_model_param1``, ``alphasat``, ``betasat``, ``bsat``, ``betacut``, ``bcut``
    """
    defaults = dict(SMHM_DEFAULTS, alphasat=1.0, betasat=0.859, bsat=10.62, betacut=-0.13, bcut=1.47)
    gal_types = ('centrals', 'satellites')

    def __init__(self, threshold=10.5, modulate_with_cenocc=True, **params):
        self.threshold = float(threshold)
        self.modulate_with_cenocc = bool(modulate_with_cenocc)
        HODModel.__init__(self, **params)

    def arguments(self):
        """the constructor arguments other than the parameters"""
        return dict(threshold=self.threshold, modulate_with_cenocc=self.modulate_with_cenocc)

    @staticmethod
    def to_halotools(cosmo, redshift, mdef, concentration_key=None, **kwargs):
        """the halotools model of the reference; halotools is not a dependency of this package"""
        raise NotImplementedError("Leauthaud11Model.to_halotools needs halotools, which is not a dependency of "
                                  "nbodykit_b200; HaloCatalog.populate evaluates the model on the GPU instead")

    def check(self):
        """ValueError unless the threshold and every parameter are finite, the scatter and bsat positive and bcut not
        negative"""
        name = type(self).__name__
        if not math.isfinite(self.threshold):
            raise ValueError("%s: the threshold must be finite (got %r)" % (name, self.threshold))
        p = self.param_dict
        for k, v in p.items():
            if not math.isfinite(v):
                raise ValueError("%s: %s must be finite (got %r)" % (name, k, v))
        if not p['scatter_model_param1'] > 0:
            raise ValueError("%s: scatter_model_param1 must be positive (got %r)" % (name, p['scatter_model_param1']))
        if not (p['bsat'] > 0 and p['bcut'] >= 0):
            raise ValueError("%s: bsat must be positive and bcut not negative (got %r, %r)"
                             % (name, p['bsat'], p['bcut']))

    def occupation(self, redshift):
        """the host-side inputs of the occupation kernel at `redshift`: dict(t, c, Msat, Mcut) (Msun/h); ValueError when
        the relation cannot be inverted or the masses are not finite"""
        p = self.param_dict
        t, c = smhm_spline(p, redshift)
        knee = 10.0 ** float(behroozi10_log_mhalo(self.threshold, p, redshift))
        msat = 1e12 * p['bsat'] * (knee / 1e12) ** p['betasat']
        mcut = 1e12 * p['bcut'] * (knee / 1e12) ** p['betacut']
        if not (math.isfinite(msat) and msat > 0 and math.isfinite(mcut)):
            raise ValueError("%s: M_sat and M_cut are not finite at redshift %r" % (type(self).__name__, redshift))
        return dict(t=t, c=c, Msat=msat, Mcut=mcut)


class Hearin15Model(Leauthaud11Model):
    r"""
    Leauthaud11Model with the Heaviside assembly bias of Hearin et al. (2016) on a secondary halo property (the
    decorated HOD of halotools' ``hearin15_model_dictionary``, with one strength each for centrals and satellites).

    Halos are binned in log10 M on a fixed grid of width ``dlog10_prim_haloprop``; within a bin they are ranked by
    ``sec_haloprop`` (ties by global row), and those with percentile above ``split`` are "upper".  Each mean N is
    shifted by the strength A (clipped to [-1, 1]) times the largest shift that keeps both halves within [0, 1]
    (centrals) or [0, inf) (satellites): upper halos get N + d, the others N - d (1 - split) / split.

    Parameters
    ----------
    threshold, modulate_with_cenocc :
        as for Leauthaud11Model
    sec_haloprop : str, optional
        the halo column that is ranked
    split : float, optional
        the percentile split, in (0, 1)
    dlog10_prim_haloprop : float, optional
        the width of the mass bins in log10 M
    **params :
        the Leauthaud11Model parameters, ``mean_occupation_centrals_assembias_param1`` and
        ``mean_occupation_satellites_assembias_param1``
    """
    defaults = dict(Leauthaud11Model.defaults, mean_occupation_centrals_assembias_param1=1.0,
                    mean_occupation_satellites_assembias_param1=0.2)

    def __init__(self, threshold=10.5, modulate_with_cenocc=True, sec_haloprop='Concentration', split=0.5,
                 dlog10_prim_haloprop=0.1, **params):
        self.sec_haloprop = str(sec_haloprop)
        self.split = float(split)
        self.dlog10_prim_haloprop = float(dlog10_prim_haloprop)
        Leauthaud11Model.__init__(self, threshold=threshold, modulate_with_cenocc=modulate_with_cenocc, **params)

    def arguments(self):
        return dict(Leauthaud11Model.arguments(self), sec_haloprop=self.sec_haloprop, split=self.split,
                    dlog10_prim_haloprop=self.dlog10_prim_haloprop)

    @staticmethod
    def to_halotools(cosmo, redshift, mdef, concentration_key=None, **kwargs):
        """the halotools model of the reference; halotools is not a dependency of this package"""
        raise NotImplementedError("Hearin15Model.to_halotools needs halotools, which is not a dependency of "
                                  "nbodykit_b200; HaloCatalog.populate evaluates the model on the GPU instead")

    def check(self):
        """Leauthaud11Model.check, and ValueError unless split is in (0, 1) and dlog10_prim_haloprop finite and
        positive"""
        Leauthaud11Model.check(self)
        if not 0 < self.split < 1:
            raise ValueError("Hearin15Model: split must be in (0, 1) (got %r)" % self.split)
        if not (math.isfinite(self.dlog10_prim_haloprop) and self.dlog10_prim_haloprop > 0):
            raise ValueError("Hearin15Model: dlog10_prim_haloprop must be finite and positive (got %r)"
                             % self.dlog10_prim_haloprop)

    def strengths(self):
        """the assembly-bias strengths of centrals and satellites, clipped to [-1, 1]"""
        p = self.param_dict
        return tuple(min(1.0, max(-1.0, p['mean_occupation_%s_assembias_param1' % g])) for g in self.gal_types)


# ---- the Jeans table ---------------------------------------------------------------------------------------------------
JEANS_S0 = -20.0          # ln y of the first node
JEANS_HS = 1.0 / 128      # node spacing in ln y
JEANS_K = 44 * 128 + 1    # nodes: ln y in [-20, 24]
_GL_X, _GL_W = numpy.polynomial.legendre.leggauss(8)


def nfw_g(y):
    """g(y) = ln(1 + y) - y / (1 + y), by its series below y = 0.1 (as the kernels evaluate it)"""
    y = numpy.asarray(y, dtype='f8')
    s = numpy.zeros_like(y)
    ys = numpy.minimum(y, 0.1)
    for m in range(16, -1, -1):
        s = s * (-ys) + float(m + 1) / float(m + 2)
    small = ys * ys * s
    with numpy.errstate(invalid='ignore', divide='ignore'):
        big = numpy.log1p(y) - y / (1.0 + y)
    return numpy.where(y < 0.1, small, big)


def _q(s):
    """the integrand of I in s = ln y: g(y) / (y^2 (1 + y)^2), so that dI / ds = -q(s)"""
    y = numpy.exp(s)
    return nfw_g(y) / (y * y * (1.0 + y) ** 2)


def _panels(a, h, n):
    """int over [a + i h, a + (i + 1) h] of q, i < n, by 8-point Gauss-Legendre"""
    left = a + numpy.arange(n) * h
    acc = numpy.zeros(n)
    for x, w in zip(_GL_X, _GL_W):
        acc += float(w) * _q(left + 0.5 * h * (1.0 + float(x)))
    return 0.5 * h * acc


_TABLE = None


def jeans_table():
    """(K, 2) float64: ln I(y) and d ln I / d ln y at ln y = JEANS_S0 + k JEANS_HS"""
    global _TABLE
    if _TABLE is None:
        s = JEANS_S0 + numpy.arange(JEANS_K) * JEANS_HS
        s1 = s[-1]
        tail = _panels(s1, JEANS_HS, int(round((64.0 - s1) / JEANS_HS))).sum()
        inner = _panels(JEANS_S0, JEANS_HS, JEANS_K - 1)
        I = numpy.empty(JEANS_K)
        I[-1] = tail
        I[:-1] = tail + numpy.cumsum(inner[::-1])[::-1]
        _TABLE = numpy.ascontiguousarray(numpy.stack([numpy.log(I), -_q(s) / I], axis=1))
    return _TABLE
