"""
Float64 NumPy/SciPy restatement of the Leauthaud11 and Hearin15 populations of DESIGN.md 4.13 (HaloCatalog.populate),
with the same counter-based draws as csrc/hod.cu, for the tests.

The occupations, the percentiles of the secondary halo property in fixed log-mass bins and the Heaviside assembly-bias
perturbation are written out here, separately from the package; the spline is scipy's InterpolatedUnivariateSpline,
evaluated by oracle/zhist_oracle.splev (FITPACK's splev in the order of its operations).  The draws, the Poisson sampler
and the galaxy placement are oracle/hod_oracle's.
"""
import contextlib

import numpy
from scipy.special import erf

from oracle import hod_oracle as ho
from oracle import zhist_oracle as zo

H_B = 0.7
LOGMS = numpy.linspace(8.5, 12.5, 100)
SMHM = dict(smhm_m0_0=10.72, smhm_m0_a=0.59, smhm_m1_0=12.35, smhm_m1_a=0.3, smhm_beta_0=0.43, smhm_beta_a=0.18,
            smhm_delta_0=0.56, smhm_delta_a=0.18, smhm_gamma_0=1.54, smhm_gamma_a=2.52, scatter_model_param1=0.2)
LEAUTHAUD11 = dict(SMHM, alphasat=1.0, betasat=0.859, bsat=10.62, betacut=-0.13, bcut=1.47)
HEARIN15 = dict(LEAUTHAUD11, mean_occupation_centrals_assembias_param1=1.0,
                mean_occupation_satellites_assembias_param1=0.2)


# ---- Behroozi et al. (2010) and its inverse ------------------------------------------------------------------------------
def log_mhalo(logms, params, z):
    """log10 M_h (Msun/h) of mean stellar mass 10^logms (Msun/h^2): X(a) = X_0 + X_a (a - 1), r = M* h^2 / 10^m0,
    log10 M_h = m1 + beta log10 r + r^delta / (1 + r^-gamma) - 1/2 (Msun), plus log10 h"""
    a = 1.0 / (1.0 + float(z))

    def X(name):
        return params['smhm_%s_0' % name] + params['smhm_%s_a' % name] * (a - 1.0)
    r = 10.0 ** numpy.asarray(logms, dtype='f8') * H_B ** 2 / 10.0 ** X('m0')
    lmh = X('m1') + X('beta') * numpy.log10(r) + r ** X('delta') / (1.0 + r ** (-X('gamma'))) - 0.5
    return lmh + numpy.log10(H_B)


def spline(params, z):
    """(t, c) of InterpolatedUnivariateSpline(log10 M_h, log10 M*, k=3) over the 100-point table"""
    from scipy.interpolate import InterpolatedUnivariateSpline
    t, c, k = InterpolatedUnivariateSpline(log_mhalo(LOGMS, params, z), LOGMS, k=3)._eval_args
    assert k == 3
    return numpy.asarray(t, 'f8'), numpy.asarray(c, 'f8')


def mean_log_mstar(mass, params, z):
    t, c = spline(params, z)
    return zo.splev(numpy.log10(numpy.asarray(mass, dtype='f8')), t, c, 0)[0]


# ---- Leauthaud et al. (2011) ---------------------------------------------------------------------------------------------
def mean_central(mass, params, z, threshold=10.5):
    logms = mean_log_mstar(mass, params, z)
    return 0.5 * (1.0 - erf((threshold - logms) / (1.4142135623730951 * params['scatter_model_param1'])))


def sat_masses(params, z, threshold=10.5):
    """(M_sat, M_cut) in Msun/h from M_knee = M_h(threshold)"""
    knee = 10.0 ** float(log_mhalo(threshold, params, z))
    return (1e12 * params['bsat'] * (knee / 1e12) ** params['betasat'],
            1e12 * params['bcut'] * (knee / 1e12) ** params['betacut'])


def mean_satellite(mass, params, z, threshold=10.5, modulate=True):
    m = numpy.asarray(mass, dtype='f8')
    msat, mcut = sat_masses(params, z, threshold)
    lam = (m / msat) ** params['alphasat'] * numpy.exp(-mcut / m)
    if modulate:
        lam = lam * mean_central(m, params, z, threshold)
    return lam


# ---- Hearin et al. (2016) assembly bias ----------------------------------------------------------------------------------
def percentiles(mass, sec, d):
    """(rank in bin + 1) / N_bin of every halo (all ranks' halos, in global row order) in its bin floor(log10 M / d),
    ranked by (sec, global row)"""
    m = numpy.asarray(mass, dtype='f8')
    b = numpy.floor(numpy.log10(m) / d)
    order = numpy.lexsort((numpy.arange(m.size), numpy.asarray(sec, dtype='f8'), b))
    pos = numpy.empty(m.size, dtype=numpy.int64)
    pos[order] = numpy.arange(m.size)
    ub, inv, cnt = numpy.unique(b, return_inverse=True, return_counts=True)
    start = numpy.cumsum(cnt) - cnt
    return (pos - start[inv] + 1).astype('f8') / cnt[inv].astype('f8')


def perturb(nb, A, p, hi, upper):
    """the mean of the upper (percentile > p) or lower halos for the baseline nb, strength A and bounds [0, hi]"""
    nb = numpy.asarray(nb, dtype='f8')
    A = min(1.0, max(-1.0, float(A)))
    r = p / (1.0 - p)
    if A >= 0:
        d = A * numpy.minimum(hi - nb, r * nb)
    else:
        d = A * numpy.minimum(nb, r * (hi - nb))
    v = numpy.where(upper, nb + d, nb - (d * (1.0 - p)) / p)
    return numpy.minimum(numpy.maximum(v, 0.0), hi)


# ---- population ----------------------------------------------------------------------------------------------------------
def means(mass, params, z, threshold=10.5, modulate=True, pct=None, split=0.5):
    """(<N_cen>, <N_sat>) of Leauthaud11, or Hearin15 when given the percentiles `pct`"""
    p = mean_central(mass, params, z, threshold)
    lam = mean_satellite(mass, params, z, threshold, modulate)
    if pct is not None:
        upper = numpy.asarray(pct) > split
        p = perturb(p, params['mean_occupation_centrals_assembias_param1'], split, 1.0, upper)
        lam = perturb(lam, params['mean_occupation_satellites_assembias_param1'], split, numpy.inf, upper)
    return p, lam


def occupy(mass, h0, params, seed, z, threshold=10.5, modulate=True, pct=None, split=0.5):
    """(N_cen, N_sat) of the halos at global rows h0 .., with hod_oracle's Bernoulli and Poisson draws"""
    m = numpy.asarray(mass, dtype='f8')
    k = ho.key(seed, 0, h0 + numpy.arange(m.size, dtype=numpy.int64))
    p, lam = means(m, params, z, threshold, modulate, pct, split)
    return (ho.uniform(k, 0) < p).astype(numpy.int64), ho.poisson(k, lam)


@contextlib.contextmanager
def _counts(ncen, nsat):
    """hod_oracle.populate with these occupation counts in place of its Zheng07 draws"""
    saved = ho.occupy
    ho.occupy = lambda *a, **kw: (ncen, nsat)
    try:
        yield
    finally:
        ho.occupy = saved


def populate(mass, radius, conc, pos, vel, box, params, seed, z, h0=0, threshold=10.5, modulate=True, rsd=1.0,
             pct=None, split=0.5):
    """the galaxy columns of one rank (global rows h0 ..), in the kernels' row order, as hod_oracle.populate; Hearin15
    when `pct` (the percentiles of these halos among all ranks') is given"""
    ncen, nsat = occupy(mass, h0, params, seed, z, threshold, modulate, pct, split)
    with _counts(ncen, nsat):
        return ho.populate(mass, radius, conc, pos, vel, box, None, seed, h0=h0, rsd=rsd)
