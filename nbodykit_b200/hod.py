"""
Halo occupation models (API of nbodykit/hod.py: HODModel, Zheng07Model) for :meth:`HaloCatalog.populate`.

The reference converts these classes to halotools models and lets halotools populate the halos on the CPU.  Here the
Zheng et al. (2007) model is evaluated by this package's own kernels (csrc/hod.cu) to the contract of DESIGN.md 4.13;
halotools is not a dependency, so :meth:`HODModel.to_halotools` raises NotImplementedError.

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

__all__ = ['HODModel', 'Zheng07Model']


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
