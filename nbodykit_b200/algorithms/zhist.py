"""
The mean number density as a function of redshift, n(z) (API of nbodykit/algorithms/zhist.py: RedshiftHistogram), on one
or several GPUs.

Contract (DESIGN.md 4.12), the reference's `run()`:

- a row goes to bin i when ``edges[i] <= z < edges[i+1]`` in float64 (``searchsorted(edges, z, 'right')`` then
  ``bincount(...)[1:-1]``): rows below the first edge, at or above the last edge and NaN are not counted;
- ``bins=None``: Scott's rule, ``h = sigma (24 sqrt(pi) / N)^(1/3)`` with the population standard deviation of all
  ranks, ``Nbins = max(1, ceil((max - min) / h))``, ``edges = min + h arange(Nbins + 1)``;
- ``bins`` an int: ``numpy.linspace(min, max, bins + 1)``; the row at the maximum sits on the last edge and is not counted;
- ``nbar = N / dV``, ``dV = 4/3 pi (R_hi^3 - R_lo^3) fsky`` with R from ``cosmo.comoving_distance``.

The kernels (csrc/zhist.cu): one pass for the count, mean, M2, min and max of the redshifts (Scott's rule and int bins),
one pass for the histogram, and one pass per :meth:`RedshiftHistogram.interpolate` for the spline.  Several GPUs: every
rank bins its own rows; the per-rank moments are gathered and merged in rank order on every rank, so that every rank
builds the same edges bit for bit, and the histograms are summed by one all-reduce.
"""
import json
import logging
import math
import numbers

import numpy
import torch

from .. import CurrentMPIComm
from .._lib import F4, F8, check, lib, stage
from ..pmesh.pm import _ptr, _stream, as_device_tensor
from .fof import _column

# scipy's InterpolatedUnivariateSpline extrapolation modes
_EXT = {0: 0, 1: 1, 2: 2, 3: 3, 'extrapolate': 0, 'zeros': 1, 'raise': 2, 'const': 3}
# explicit edges within this fraction of a bin of an arithmetic sequence are binned by the arithmetic guess
_EVEN_TOL = 1e-3


def _code(t):
    return F4 if t.dtype == torch.float32 else F8


class RedshiftHistogram(object):
    r"""
    Compute the mean number density as a function of redshift :math:`n(z)` from an input CatalogSource of particles,
    in :math:`(\mathrm{Mpc}/h)^{-3}`.  Runs on construction; :meth:`run` computes it again.

    Parameters
    ----------
    source : CatalogSource
        the source of particles holding the redshift column to histogram
    fsky : float
        the sky area fraction (positive, finite), used in the volume of the redshift shells
    cosmo : Cosmology
        converts redshift into comoving distance; any object with ``comoving_distance(z)``
    bins : int or sequence of scalars, optional
        an int: that many equal-width bins from the smallest to the largest redshift of all ranks, as
        ``numpy.linspace(min, max, bins + 1)``.  The row at the largest redshift sits on the last edge and, as every row
        at or above the last edge, is not counted.  A sequence: the bin edges, rightmost included (1-D, at least two,
        finite, strictly increasing, above -1).  None (default): Scott's rule over the redshifts of all ranks
    redshift : str, optional
        the name of the redshift column
    weight : str, optional
        the name of a weight column to histogram instead of counting rows

    Scott's rule and int bins need finite redshifts and a non-empty catalogue with some spread; they raise
    ``ValueError`` on every rank otherwise.

    Attributes (the same on every rank)
    -----------------------------------
    bin_edges, bin_centers : numpy.ndarray
        the edges of the redshift bins and their midpoints
    dV : numpy.ndarray
        the volume of each redshift shell in :math:`(\mathrm{Mpc}/h)^3`
    nbar : numpy.ndarray
        float64: the counts (exact integers) or weight sums of each bin over dV
    attrs : dict
        ``edges``, ``fsky``, ``redshift``, ``weight`` and ``cosmo`` (``cosmo.pars`` for a :class:`Cosmology`,
        ``dict(cosmo)`` for a mapping, else None)
    """
    logger = logging.getLogger('RedshiftHistogram')

    def __init__(self, source, fsky, cosmo, bins=None, redshift='Redshift', weight=None):
        for col in [redshift, weight]:
            if col is not None and col not in source:
                raise ValueError("'%s' column missing from input source in RedshiftHistogram" % col)
        if not (numpy.isscalar(fsky) and not isinstance(fsky, (str, bytes)) and numpy.isfinite(fsky) and fsky > 0):
            raise ValueError("RedshiftHistogram: fsky must be a positive finite number (got %r)" % (fsky,))
        if not callable(getattr(cosmo, 'comoving_distance', None)):
            raise ValueError("RedshiftHistogram: cosmo must provide comoving_distance(z)")

        self.comm = source.comm
        self.source = source
        self.cosmo = cosmo

        z = None
        if bins is None:
            z = _column(source, redshift, None)
            h, bins = scotts_bin_width(z, self.comm)
            if self.comm.rank == 0:
                self.logger.info("using Scott's rule to determine optimal binning; h = %.2e, N_bins = %d" % (h, len(bins) - 1))
        elif numpy.isscalar(bins):
            if isinstance(bins, (bool, numpy.bool_)) or not isinstance(bins, numbers.Integral) or bins < 1:
                raise ValueError("RedshiftHistogram: an int `bins` must be a positive integer (got %r)" % (bins,))
            if self.comm.rank == 0:
                self.logger.info("computing %d equally spaced bins" % bins)
            z = _column(source, redshift, None)
            m = global_moments(z, self.comm)
            _check_moments(m, "equally spaced bins")
            bins = numpy.linspace(m[3], m[4], int(bins) + 1, endpoint=True)
        else:
            bins = _check_edges(bins)

        self.attrs = {}
        self.attrs['edges'] = bins
        self.attrs['fsky'] = fsky
        self.attrs['redshift'] = redshift
        self.attrs['weight'] = weight
        self.attrs['cosmo'] = _cosmo_attr(cosmo)

        self._run(z)

    def run(self):
        """
        Compute the histogram.  Adds :attr:`bin_edges`, :attr:`bin_centers`, :attr:`dV` and :attr:`nbar`, the same on
        every rank.
        """
        self._run(None)

    def _run(self, z):
        edges = numpy.asarray(self.attrs['edges'], dtype='f8')
        if z is None:
            z = _column(self.source, self.attrs['redshift'], None)
        w = None
        if self.attrs['weight'] is not None:
            w = _column(self.source, self.attrs['weight'], z.device)
            if self.comm.rank == 0:
                self.logger.info("computing histogram using weights from '%s' column" % self.attrs['weight'])
        N = histogram(z, w, edges, self.comm)

        if self.comm.rank == 0:
            self.logger.info("using cosmology %s to compute volume in units of (Mpc/h)^3" % str(self.cosmo))
            self.logger.info("sky fraction used in volume calculation: %.4f" % self.attrs['fsky'])
        R_hi = numpy.asarray(self.cosmo.comoving_distance(edges[1:]), dtype='f8')
        R_lo = numpy.asarray(self.cosmo.comoving_distance(edges[:-1]), dtype='f8')
        dV = (4. / 3.) * numpy.pi * (R_hi ** 3 - R_lo ** 3) * self.attrs['fsky']

        self.bin_edges = edges
        self.bin_centers = 0.5 * (edges[:-1] + edges[1:])
        self.dV = dV
        self.nbar = 1. * N / dV

    def interpolate(self, z, ext='zeros'):
        """
        Interpolate n(z) with scipy's ``InterpolatedUnivariateSpline(bin_centers, nbar, ext=ext)``, a cubic
        interpolating spline, evaluated on the GPU.  The interpolation acts as a band-pass filter, removing small-scale
        fluctuations of the estimate.

        Parameters
        ----------
        z : array_like, Column or torch.Tensor
            redshift, float32 or float64
        ext : 'extrapolate' (0), 'zeros' (1), 'raise' (2) or 'const' (3)
            how to treat redshifts outside ``[bin_centers[0], bin_centers[-1]]``.  'raise' raises ``ValueError`` on
            every rank when any rank has such a redshift

        Returns
        -------
        n : float64; a torch tensor on the device of a tensor (or tensor-backed Column) input, else a NumPy array of
            the shape of z
        """
        try:
            code = _EXT[ext]
        except (KeyError, TypeError):
            raise ValueError("Unknown extrapolation mode %s." % (ext,))
        t, c = self._spline()
        if hasattr(z, 'materialize'):
            z = z.materialize()
        elif hasattr(z, 'compute'):
            z = z.compute()
        as_tensor = isinstance(z, torch.Tensor)
        shape = tuple(z.shape) if as_tensor else numpy.shape(z)
        zt = as_device_tensor(z if as_tensor else numpy.asarray(z), device=t.device).reshape(-1)
        if zt.dtype not in (torch.float32, torch.float64):
            zt = zt.to(torch.float64)
        zt = zt.contiguous()
        n = int(zt.shape[0])
        out = torch.empty(n, dtype=torch.float64, device=t.device)
        outside = torch.zeros(1, dtype=torch.int64, device=t.device)
        with stage("zh_spline"):
            check(lib().nbk_zh_spline(_ptr(zt), _code(zt), n, _ptr(t), int(t.shape[0]), _ptr(c), code, _ptr(out),
                                      _ptr(outside), _stream()), "nbk_zh_spline")
        if code == 2 and int(self.comm.allreduce(int(outside.item()))) > 0:
            raise ValueError("Found x value not in the domain")
        out = out.reshape(shape)
        if as_tensor:
            return out.to(z.device)
        return out.cpu().numpy()

    def _spline(self):
        """the knots and coefficients of the spline of nbar at the bin centers, on the device (built from scipy on the
        host, once per histogram)"""
        key = (numpy.asarray(self.bin_centers, 'f8').tobytes(), numpy.asarray(self.nbar, 'f8').tobytes())
        cached = getattr(self, '_spline_cache', None)
        if cached is not None and cached[0] == key:
            return cached[1]
        from scipy.interpolate import InterpolatedUnivariateSpline
        x = numpy.asarray(self.bin_centers, dtype='f8')
        if x.ndim != 1 or len(x) < 4:
            raise ValueError("RedshiftHistogram.interpolate needs at least 4 bins for a cubic spline (got %d)" % x.size)
        t, c, k = InterpolatedUnivariateSpline(x, numpy.asarray(self.nbar, dtype='f8'))._eval_args
        assert k == 3
        dev = torch.device('cuda', torch.cuda.current_device())
        tc = (torch.from_numpy(numpy.ascontiguousarray(t, 'f8')).to(dev),
              torch.from_numpy(numpy.ascontiguousarray(c, 'f8')).to(dev))
        self._spline_cache = (key, tc)
        return tc

    def __getstate__(self):
        state = dict(bin_edges=self.bin_edges,
                     bin_centers=self.bin_centers,
                     dV=self.dV,
                     nbar=self.nbar,
                     attrs=self.attrs)
        return state

    def __setstate__(self, state):
        self.__dict__.update(state)

    def save(self, output):
        """Save the result to ``output`` as JSON (rank 0 writes)."""
        from ..utils import JSONEncoder
        if self.comm.rank == 0:
            self.logger.info('histogram done; saving result to %s' % output)
            with open(output, 'w') as ff:
                json.dump(self.__getstate__(), ff, cls=JSONEncoder)

    @classmethod
    @CurrentMPIComm.enable
    def load(cls, output, comm=None):
        """Load a result written by :meth:`save` (rank 0 reads, every rank gets it)."""
        from ..utils import JSONDecoder
        if comm.rank == 0:
            with open(output, 'r') as ff:
                state = json.load(ff, cls=JSONDecoder)
        else:
            state = None
        state = comm.bcast(state)
        self = object.__new__(cls)
        self.__setstate__(state)
        self.comm = comm
        return self


def _cosmo_attr(cosmo):
    from ..cosmology import Cosmology
    if isinstance(cosmo, Cosmology):
        return dict(cosmo.pars)
    try:
        return dict(cosmo)
    except (TypeError, ValueError):
        return None


def _check_edges(bins):
    e = numpy.asarray(bins)
    if e.dtype.kind not in 'biuf':
        raise ValueError("RedshiftHistogram: bin edges must be numbers")
    e = e.astype('f8')
    if e.ndim != 1 or len(e) < 2:
        raise ValueError("RedshiftHistogram: bin edges must be 1-D with at least two entries")
    if not numpy.isfinite(e).all():
        raise ValueError("RedshiftHistogram: bin edges must be finite")
    if not (numpy.diff(e) > 0).all():
        raise ValueError("RedshiftHistogram: bin edges must be strictly increasing")
    if not (e[0] > -1):
        raise ValueError("RedshiftHistogram: bin edges must be above -1")
    return e


def _merge(a, b):
    """Chan's rule on (count, mean, M2, min, max, non-finite) tuples, as the kernel's"""
    bad = a[5] + b[5]
    if b[0] == 0:
        return a[:5] + (bad,)
    if a[0] == 0:
        return b[:5] + (bad,)
    n = a[0] + b[0]
    d = b[1] - a[1]
    fb = b[0] / n
    return (n, a[1] + d * fb, (a[2] + b[2]) + (d * d) * (a[0] * fb), min(a[3], b[3]), max(a[4], b[4]), bad)


def local_moments(z):
    """(count, mean, M2, min, max, non-finite count) of the finite rows of a device column, as Python floats"""
    n = int(z.shape[0])
    if n == 0:
        return (0.0, 0.0, 0.0, math.inf, -math.inf, 0.0)
    L = lib()
    partial = torch.empty(int(L.nbk_zh_partials()) * 6, dtype=torch.float64, device=z.device)
    out = torch.empty(6, dtype=torch.float64, device=z.device)
    check(L.nbk_zh_moments(_ptr(z), _code(z), n, _ptr(partial), _ptr(out), _stream()), "nbk_zh_moments")
    return tuple(float(v) for v in out.cpu().tolist())


def global_moments(z, comm):
    """the moments of all ranks, merged in rank order on every rank (the same bits everywhere)"""
    with stage("zh_moments"):
        parts = comm.allgather(local_moments(z))
    m = parts[0]
    for p in parts[1:]:
        m = _merge(m, p)
    return m


def _check_moments(m, what):
    if m[5] > 0:
        raise ValueError("RedshiftHistogram: %d non-finite redshifts; %s need finite redshifts" % (int(m[5]), what))
    if m[0] == 0:
        raise ValueError("RedshiftHistogram: the catalogue is empty; %s need redshifts" % what)
    if not (m[4] > m[3]) or not (m[2] > 0):
        raise ValueError("RedshiftHistogram: the redshifts have zero spread; %s need some" % what)


def scotts_bin_width(z, comm):
    r"""
    The histogram bin width of Scott's rule over the redshifts of all ranks, and the edges from the smallest redshift:

    .. math::

        h = \sigma \sqrt[3]{\frac{24 \sqrt{\pi}}{n}}

    A collective operation.  Raises ``ValueError`` on every rank for non-finite redshifts, an empty catalogue or
    redshifts with zero spread.
    """
    m = global_moments(z, comm)
    _check_moments(m, "Scott's rule bins")
    csize, _, m2, minval, maxval, _ = m
    sigma = (m2 / csize) ** 0.5
    dx = sigma * (24. * numpy.sqrt(numpy.pi) / csize) ** (1. / 3)
    if not (dx > 0):
        raise ValueError("RedshiftHistogram: the redshifts have zero spread; Scott's rule bins need some")
    Nbins = numpy.ceil((maxval - minval) * 1. / dx)
    Nbins = int(max(1, Nbins))
    edges = minval + dx * numpy.arange(Nbins + 1)
    return dx, edges


def _inverse_width(edges):
    """1 / the bin width when the edges are evenly spaced (within _EVEN_TOL of a bin), else 0"""
    nb = len(edges) - 1
    h = (edges[-1] - edges[0]) / nb
    if not (h > 0):
        return 0.0
    dev = numpy.abs(edges - (edges[0] + h * numpy.arange(nb + 1))).max()
    return 1.0 / h if dev <= _EVEN_TOL * h else 0.0


def histogram(z, w, edges, comm):
    """the counts (float64 of exact integers) or weight sums per bin of device redshifts z (and weights w) over all
    ranks: a row goes to bin i when edges[i] <= z < edges[i+1]"""
    dev = z.device
    nb = len(edges) - 1
    n = int(z.shape[0])
    e = torch.from_numpy(numpy.ascontiguousarray(edges, 'f8')).to(dev)
    counts = torch.zeros(nb, dtype=torch.int64, device=dev)
    sums = torch.zeros(nb, dtype=torch.float64, device=dev) if w is not None else None
    if w is not None and int(w.shape[0]) != n:
        raise ValueError("RedshiftHistogram: the weight column has %d rows, the redshifts %d" % (int(w.shape[0]), n))
    with stage("zh_bin"):
        check(lib().nbk_zh_bin(_ptr(z), _code(z), _ptr(w), _code(w) if w is not None else 0, n, _ptr(e), nb,
                               _inverse_width(edges), _ptr(counts), _ptr(sums), _stream()), "nbk_zh_bin")
    with stage("zh_reduce"):
        if comm.size > 1:
            counts = comm.allreduce_tensor(counts)
            if sums is not None:
                sums = comm.allreduce_tensor(sums)
        out = (sums if sums is not None else counts).cpu().numpy()
    return out.astype('f8')
