"""
TEST INFRASTRUCTURE -- a float64 NumPy / SciPy restatement of the RedshiftHistogram contract (DESIGN.md 4.12).

- Scott's rule: mean = sum / N, sigma = sqrt(sum((z - mean)^2) / N), h = sigma (24 sqrt(pi) / N)^(1/3),
  Nbins = max(1, ceil((max - min) / h)), edges = min + h arange(Nbins + 1);
- int bins: linspace(min, max, bins + 1);
- a row goes to bin i when edges[i] <= z < edges[i+1] (z widened to float64); NaN and rows outside are not counted;
- nbar = N / dV, dV = 4/3 pi (R_hi^3 - R_lo^3) fsky;
- interpolate: scipy's InterpolatedUnivariateSpline(bin_centers, nbar, ext), and `splev`, the same (t, c) evaluated by a
  vectorised restatement of FITPACK's splev / fpbspl in the order of its operations.

`with_zhist_norms` runs the n(z) part of the reference's test_conv_power.py::test_with_zhist on this package's
MPIRandomState streams and Planck15 and returns the FKP normalisations it implies.
"""
import numpy

EXT = {0: 0, 1: 1, 2: 2, 3: 3, 'extrapolate': 0, 'zeros': 1, 'raise': 2, 'const': 3}


def scott_edges(z):
    """(h, edges) of Scott's rule over the float64 redshifts z"""
    z = numpy.asarray(z, dtype='f8')
    N = z.size
    mean = z.sum() / N
    sigma = (((z - mean) ** 2).sum() / N) ** 0.5
    h = sigma * (24. * numpy.sqrt(numpy.pi) / N) ** (1. / 3)
    nbins = int(max(1, numpy.ceil((z.max() - z.min()) / h)))
    return h, z.min() + h * numpy.arange(nbins + 1)


def int_edges(z, bins):
    z = numpy.asarray(z, dtype='f8')
    return numpy.linspace(z.min(), z.max(), bins + 1)


def counts(z, edges, w=None):
    """per bin: the number of rows (or the sum of their weights, float64) with edges[i] <= z < edges[i+1]"""
    z = numpy.asarray(z).astype('f8')
    edges = numpy.asarray(edges, dtype='f8')
    nb = len(edges) - 1
    idx = numpy.searchsorted(edges, z, side='right') - 1
    ok = (idx >= 0) & (idx < nb)
    if w is None:
        return numpy.bincount(idx[ok], minlength=nb).astype('f8')
    return numpy.bincount(idx[ok], weights=numpy.asarray(w).astype('f8')[ok], minlength=nb)


def shell_volumes(edges, fsky, cosmo):
    R_hi = numpy.asarray(cosmo.comoving_distance(edges[1:]), dtype='f8')
    R_lo = numpy.asarray(cosmo.comoving_distance(edges[:-1]), dtype='f8')
    return (4. / 3.) * numpy.pi * (R_hi ** 3 - R_lo ** 3) * fsky


def zhist(z, fsky, cosmo, bins=None, w=None):
    """dict(bin_edges, bin_centers, dV, nbar, N) of one catalogue"""
    if bins is None:
        edges = scott_edges(z)[1]
    elif numpy.isscalar(bins):
        edges = int_edges(z, bins)
    else:
        edges = numpy.asarray(bins, dtype='f8')
    N = counts(z, edges, w)
    dV = shell_volumes(edges, fsky, cosmo)
    return dict(bin_edges=edges, bin_centers=0.5 * (edges[:-1] + edges[1:]), dV=dV, nbar=1. * N / dV, N=N)


def spline(centers, nbar):
    """(t, c) of scipy's cubic interpolating spline through (centers, nbar)"""
    from scipy.interpolate import InterpolatedUnivariateSpline
    t, c, k = InterpolatedUnivariateSpline(centers, nbar)._eval_args
    assert k == 3
    return numpy.asarray(t, 'f8'), numpy.asarray(c, 'f8')


def interpolate(z, centers, nbar, ext='zeros'):
    """scipy's InterpolatedUnivariateSpline(centers, nbar, ext=ext)(z)"""
    from scipy.interpolate import InterpolatedUnivariateSpline
    return InterpolatedUnivariateSpline(centers, nbar, ext=ext)(z)


def splev(z, t, c, ext):
    """FITPACK's splev for k = 3 restated: (values, rows outside [t[3], t[-4]]); ext 2 returns the extrapolated values"""
    k = 3
    ext = EXT[ext]
    x = numpy.atleast_1d(numpy.asarray(z).astype('f8')).ravel().copy()
    nt = len(t)
    tb, te = t[k], t[nt - k - 1]
    oob = (x < tb) | (x > te)
    if ext == 3:
        x = numpy.where(x < tb, tb, numpy.where(x > te, te, x))
    # the largest l in [k, nt - k - 2] with t[l] <= x (k when none; NaN ends at k as well, its value is NaN anyway)
    l = numpy.clip(numpy.searchsorted(t, x, side='right') - 1, k, nt - k - 2)
    l = numpy.where(numpy.isnan(x), k, l)
    h = [numpy.ones_like(x)] + [numpy.zeros_like(x) for _ in range(k)]
    for j in range(1, k + 1):
        hh = [v.copy() for v in h[:j]]
        h[0] = numpy.zeros_like(x)
        for i in range(1, j + 1):
            tli, tlj = t[l + i], t[l + i - j]
            same = tli == tlj
            with numpy.errstate(divide='ignore', invalid='ignore'):
                f = hh[i - 1] / (tli - tlj)
                hi1 = h[i - 1] + f * (tli - x)
                hi = f * (x - tlj)
            h[i - 1] = numpy.where(same, h[i - 1], hi1)
            h[i] = numpy.where(same, 0.0, hi)
    sp = numpy.zeros_like(x)
    for j in range(k + 1):
        sp = sp + c[l - k + j] * h[j]
    if ext == 1:
        sp = numpy.where(oob, 0.0, sp)
    return sp, int(oob.sum())


# the reference's test_conv_power.py::test_with_zhist
NDATA = 1000
FSKY = 0.15
DATA_NORM = 0.000388338522187
RANDOMS_NORM = 0.000395808747269


def make_redshifts(seed, n):
    """the z column of the reference test's make_sources: the first draw of RandomCatalog(n, seed).rng"""
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.mpirng import MPIRandomState
    return MPIRandomState(SelfComm(), seed=seed, size=n).normal(loc=0.5, scale=0.1)


def with_zhist_norms(cosmo=None):
    """(data.norm, randoms.norm, data NZ, randoms NZ) of test_with_zhist: n(z) of the randoms by Scott's rule, NZ =
    interpolate(z) alpha, and the FKP normalisations with unit weights: sum(NZ_data) and alpha sum(NZ_randoms)"""
    if cosmo is None:
        from nbodykit_b200.cosmology import Planck15 as cosmo
    zd = make_redshifts(42, NDATA)
    zr = make_redshifts(84, NDATA * 10)
    r = zhist(zr, FSKY, cosmo)
    alpha = 1.0 * len(zd) / len(zr)
    nz_r = interpolate(zr, r['bin_centers'], r['nbar']) * alpha
    nz_d = interpolate(zd, r['bin_centers'], r['nbar']) * alpha
    return float(nz_d.sum()), float(nz_r.sum()) * alpha, nz_d, nz_r
