"""
Multipoles of the isotropic three-point correlation function in a simulation box (API of
nbodykit/algorithms/threeptcf.py: SimulationBox3PCF) on one or several GPUs.

The reference enumerates the neighbours of every primary with kdcount in Python; here it is csrc/threeptcf.cu, under a
contract stated in double precision (DESIGN.md 4.7): per-axis d = x_j - x_p from the positions as stored (periodic:
wrapped with `pos % L` in their own dtype, then d > L/2 -> d - L, d <= -L/2 -> d + L), r = sqrt((dx^2 + dy^2) + dz^2),
radial bin k holding e_k < r <= e_{k+1} with r > 0, and

    zeta_l(b1, b2) = (2l + 1) / (16 pi^2) sum_p w_p sum_{j in b1} sum_{k in b2} w_j w_k P_l(u_pj . u_pk)

(the sum includes j = k).  The kernel evaluates it through the spherical-harmonic moments of each primary's neighbours
(the addition theorem), with the coefficient table built here in exact rational arithmetic.  The catalogue is sorted
into cells of side >= r_max / 2 with the FOF cell machinery (csrc/fof.cu), and the neighbours are walked on the stencil
of the pair counts (csrc/pc_cells.cuh).

Several GPUs: x slabs of the box, as for the pair counts: every primary is handled on the rank whose slab holds it, with
copies of the rows within r_max of a remote slab as its secondaries; zeta, the pair counts and the candidate count are
combined in one all-reduce.
"""
import logging
import math
from decimal import Decimal, localcontext
from fractions import Fraction

import numpy
import torch

from .. import CurrentMPIComm
from .._lib import check, darr, i32arr, iarr, lib, stage
from ..binned_statistic import BinnedStatistic
from ..pmesh.pm import _ptr, _stream
from .fof import _column
from .paircount import (_CELLS_PER_SMAX, _Cells, _check_rows, _verify_columns, _verify_sources, slab_route,
                        weight_column)


def max_ell():
    """the largest pole the kernel computes"""
    return int(lib().nbk_threeptcf_max_ell())


def max_bins():
    """the largest number of radial bins the kernel computes"""
    return int(lib().nbk_threeptcf_max_bins())


def _legendre(ell):
    """the coefficients of P_ell(z) in powers of z, as Fractions (index = power)"""
    c = [Fraction(0)] * (ell + 1)
    for k in range(ell // 2 + 1):
        c[ell - 2 * k] = Fraction((-1) ** k * math.comb(ell, k) * math.comb(2 * ell - 2 * k, ell), 2 ** ell)
    return c


def q_poly(ell, m):
    r"""the coefficients (index = power of z) of Q_lm(z) = (-1)^m d^m P_l / dz^m, so that
    :math:`Y_{lm}(\hat u) = N_{lm} (u_x + i u_y)^m Q_{lm}(u_z)` with
    :math:`N_{lm}^2 = (2l + 1) / (4 \pi) \, (l - m)! / (l + m)!` (Condon-Shortley phase); exact Fractions"""
    p = _legendre(ell)
    out = [Fraction(0)] * (ell - m + 1)
    for n in range(m, ell + 1):
        out[n - m] = (-1) ** m * p[n] * Fraction(math.factorial(n), math.factorial(n - m))
    return out


def coefficient_table(L):
    r"""the [(L+1)(L+2)/2][L+1] table T of the kernel: a_lm = sum_k T[lm][k] M_{m,k}, lm = off(m) + l - m with
    off(m) = m (L + 1) - m (m - 1) / 2, equal to :math:`\sqrt{4\pi}\, N_{lm}` times the coefficient of
    :math:`u_z^k` in Q_lm.  Each entry is sign(q) sqrt(q^2 (2l + 1) (l - m)! / (l + m)!) with the radicand an exact
    rational, evaluated to 40 digits and rounded once to double."""
    nmom = (L + 1) * (L + 2) // 2
    T = numpy.zeros((nmom, L + 1))
    with localcontext() as ctx:
        ctx.prec = 40
        for m in range(L + 1):
            off = m * (L + 1) - m * (m - 1) // 2
            for ell in range(m, L + 1):
                norm2 = Fraction((2 * ell + 1) * math.factorial(ell - m), math.factorial(ell + m))
                for k, q in enumerate(q_poly(ell, m)):
                    if q == 0:
                        continue
                    r = q * q * norm2
                    v = (Decimal(r.numerator) / Decimal(r.denominator)).sqrt()
                    T[off + ell - m, k] = float(v) if q > 0 else -float(v)
    return T


def _check_edges(edges):
    e = numpy.asarray(edges, dtype='f8')
    if e.ndim != 1 or len(e) < 2 or not numpy.isfinite(e).all() or not (numpy.diff(e) > 0).all() or e[0] < 0:
        raise ValueError("3PCF: edges must be a 1-D array of at least two finite, strictly increasing values, the first "
                         ">= 0")
    if len(e) - 1 > max_bins():
        raise ValueError("3PCF: %d radial bins; at most %d are supported (poles up to l = %d)"
                         % (len(e) - 1, max_bins(), max_ell()))
    return e


def _check_poles(poles):
    try:
        p = list(poles)
    except TypeError:
        raise ValueError("3PCF: poles must be a list of non-negative integers")
    if len(p) == 0:
        raise ValueError("3PCF: poles must be a non-empty list of non-negative integers")
    for v in p:
        if isinstance(v, (bool, numpy.bool_)) or not isinstance(v, (int, numpy.integer)) or v < 0:
            raise ValueError("3PCF: poles must be non-negative integers (got %r)" % (v,))
    p = [int(v) for v in p]
    if len(set(p)) != len(p):
        raise ValueError("3PCF: poles must be unique (got %s)" % p)
    if max(p) > max_ell():
        raise ValueError("3PCF: pole %d is above the largest supported, l = %d (with at most %d radial bins)"
                         % (max(p), max_ell(), max_bins()))
    return p


def count_triplets(pos1, w1, pos2, w2, edges, poles, periodic, box):
    """zeta_l(b1, b2) of the primaries pos1 against the secondaries pos2 on this device, per the contract of DESIGN.md
    4.7, without the factor 1 / (16 pi^2) and with only b1 <= b2 filled.  pos: (n, 3) float32 / float64 device
    tensors; w: float64 (n,).  Returns device tensors (zeta f64 [len(poles)][nb][nb], npairs int64 [nb]) and the number
    of candidate pairs tested."""
    dev = pos1.device
    e = numpy.asarray(edges, dtype='f8')
    nb = len(e) - 1
    L = max(poles)
    zeta = torch.zeros((len(poles), nb, nb), dtype=torch.float64, device=dev)
    npairs = torch.zeros(nb, dtype=torch.int64, device=dev)
    cand = torch.zeros(1, dtype=torch.int64, device=dev)
    n1, n2 = int(pos1.shape[0]), int(pos2.shape[0])
    if n1 == 0 or n2 == 0:
        return zeta, npairs, 0
    box = numpy.asarray(box, 'f8')
    if periodic:
        gbox = box
        origin = numpy.zeros(3)
    else:
        lo = torch.minimum(pos1.min(0).values.double(), pos2.min(0).values.double()).cpu().numpy()
        hi = torch.maximum(pos1.max(0).values.double(), pos2.max(0).values.double()).cpu().numpy()
        origin = lo
        gbox = numpy.where(hi > lo, hi - lo, 1.0)
    rmax = float(e[-1])
    ncell = [int(min(max(1, math.floor(Lx * _CELLS_PER_SMAX / (rmax * (1 + 1e-4)))), 1 << 20)) for Lx in gbox]
    # a row may sit outside its cell by the rounding of its cell index, or by L_f4 - L_f8 when an f4 position wraps to L
    tol = 4e-7 * (gbox + numpy.abs(origin))
    with stage("threeptcf_cells"):
        c2 = _Cells(pos2, w2, periodic, gbox, origin, ncell)
        c1 = c2 if pos1 is pos2 and w1 is w2 else _Cells(pos1, w1, periodic, gbox, origin, ncell)
        first, ckey, nchunks = c1.chunks(int(lib().nbk_threeptcf_chunk_rows()))
    T = numpy.ascontiguousarray(coefficient_table(L))
    work = torch.empty(len(e) + T.size, dtype=torch.float64, device=dev)
    with stage("threeptcf_count"):
        check(lib().nbk_threeptcf(_ptr(c1.pos), _ptr(c1.w), _ptr(first), _ptr(ckey), nchunks, _ptr(c2.pos), _ptr(c2.w),
                                  _ptr(c2.cell_start), _ptr(c2.cell_key), c2.ncells, int(periodic), darr(gbox), iarr(ncell),
                                  darr(tol), darr(e), len(e), i32arr(poles), len(poles), darr(T.ravel()), _ptr(work),
                                  _ptr(zeta), _ptr(npairs), _ptr(cand), _stream()), "nbk_threeptcf")
    return zeta, npairs, int(cand.item())


class SimulationBox3PCF(object):
    r"""
    The multipoles :math:`\zeta_\ell(r_1, r_2)` of the isotropic three-point correlation function of objects in a
    simulation box (Slepian and Eisenstein, MNRAS 454, 4142 (2015)), on one or several GPUs.  Runs on construction.

    Parameters
    ----------
    source : CatalogSource
        the catalogue; it provides both the primaries and the secondaries
    poles : list of int
        the multipoles to compute, distinct, from 0 up to :func:`max_ell` (10)
    edges : array_like
        the radial bin edges, finite, strictly increasing, the first >= 0; at most :func:`max_bins` (32) bins.  Bin k
        holds the separations e_k < r <= e_{k+1}; a pair at r = 0 never counts
    BoxSize : float, 3-vector, optional
        the box; if not given, ``source.attrs['BoxSize']``.  Periodic boxes need not be cubic
    periodic : bool, optional
        minimum-image separations; then ``max(edges)`` may not exceed half the smallest side
    weight : str, optional
        the weight column
    position : str, optional
        the position column

    At most 2^31 - 1 rows per rank.

    Attributes
    ----------
    poles : BinnedStatistic
        dims ``['r1', 'r2']``, one variable ``corr_<l>`` per pole, in the order given:
        :math:`\zeta_\ell = \frac{2\ell + 1}{16\pi^2} \sum_p w_p \sum_{j \in b_1} \sum_{k \in b_2} w_j w_k
        P_\ell(\hat u_{pj} \cdot \hat u_{pk})`, which is the reference's normalisation (the C++ code of the reference's
        test data differs by :math:`(4\pi)^2 / (2\ell + 1)`)
    npairs : numpy.ndarray
        u8 per radial bin: the ordered (primary, secondary) pairs in the bin
    candidates : int
        the (primary, secondary) pairs the kernel tested
    """
    logger = logging.getLogger('SimulationBox3PCF')

    def __init__(self, source, poles, edges, BoxSize=None, periodic=True, weight='Weight', position='Position'):
        BoxSize = _verify_sources(source, None, BoxSize, [position, weight])
        p = _check_poles(poles)
        _check_edges(edges)
        self.source = source
        self.comm = source.comm
        self.attrs = {}
        self.attrs['poles'] = p
        self.attrs['edges'] = edges
        self.attrs['BoxSize'] = BoxSize
        self.attrs['periodic'] = periodic
        self.attrs['weight'] = weight
        self.attrs['position'] = position
        if periodic:
            if numpy.amax(edges) > 0.5 * BoxSize.min():
                raise ValueError("periodic pair counts cannot be computed for Rmax > BoxSize/2")
        self.poles = self.run()

    def _weights(self):
        return weight_column(self.source, self.attrs['weight'])

    def _rows(self):
        """(positions, float64 weights) of the catalogue on the device"""
        pos = _column(self.source, self.attrs['position'], None)
        if pos.ndim != 2 or pos.shape[1] != 3:
            raise ValueError("3PCF: Position must have shape (n, 3)")
        return pos, self._weights()

    def run(self, pedantic=False):
        """compute the multipoles; sets and returns :attr:`poles`, and sets :attr:`npairs` and :attr:`candidates`.
        ``pedantic`` is accepted for the reference's signature and has no effect: the reference's pedantic run only
        changes how its tree enumeration is batched, which does not change the result"""
        comm = self.comm
        attrs = self.attrs
        periodic = bool(attrs['periodic'])
        poles = _check_poles(attrs['poles'])
        e = _check_edges(attrs['edges'])
        pos, w = self._rows()
        _check_rows(int(pos.shape[0]), "the catalogue")
        box = numpy.asarray(attrs['BoxSize'], 'f8') if periodic else None
        rmax = float(e[-1])
        with stage("threeptcf_route"):
            if comm.size > 1:
                pos1, w1, pos2, w2 = slab_route(comm, pos, w, pos, w, periodic, box, rmax)
                _check_rows(int(pos1.shape[0]), "primaries after routing")
                _check_rows(int(pos2.shape[0]), "secondaries after routing")
            else:
                pos1, w1, pos2, w2 = pos, w, pos, w
        zeta, npairs, cand = count_triplets(pos1, w1, pos2, w2, e, poles, periodic, box)
        with stage("threeptcf_reduce"):
            zeta, npairs, cand = self._reduce(zeta, npairs, cand)
        self.npairs = npairs
        self.candidates = cand
        nb = len(e) - 1
        iu = numpy.triu_indices(nb, 1)
        zeta[:, iu[1], iu[0]] = zeta[:, iu[0], iu[1]]
        zeta /= 16. * numpy.pi ** 2
        data = numpy.empty((nb, nb), dtype=[('corr_%d' % ell, 'f8') for ell in poles])
        for i, ell in enumerate(poles):
            data['corr_%d' % ell] = zeta[i]
        self.poles = BinnedStatistic(['r1', 'r2'], [attrs['edges'], attrs['edges']], data)
        return self.poles

    def _reduce(self, zeta, npairs, cand):
        """host arrays of zeta, npairs and the candidate count summed over ranks in one f64 all-reduce (the counts as
        two exact 32-bit halves)"""
        comm = self.comm
        if comm.size == 1:
            return zeta.cpu().numpy(), npairs.cpu().numpy().astype('u8'), int(cand)
        c = torch.cat([npairs, torch.tensor([cand], dtype=torch.int64, device=npairs.device)])
        packed = torch.cat([(c & 0xffffffff).to(torch.float64), (c >> 32).to(torch.float64), zeta.reshape(-1)])
        comm.allreduce_tensor(packed, "sum")
        k = c.shape[0]
        tot = (packed[k:2 * k].round().to(torch.int64) << 32) + packed[:k].round().to(torch.int64)
        nb = npairs.shape[0]
        return (packed[2 * k:].reshape(zeta.shape).cpu().numpy(), tot[:nb].cpu().numpy().astype('u8'),
                int(tot[nb].item()))

    # ------------------------------------------------------------------------------------------------------------------
    def __getstate__(self):
        return {'poles': self.poles.data, 'attrs': self.attrs}

    def __setstate__(self, state):
        self.__dict__.update(state)
        self.poles = BinnedStatistic(['r1', 'r2'], [self.attrs['edges']] * 2, self.poles)

    def save(self, output):
        """save the :attr:`poles` result as JSON (``{'poles': ..., 'attrs': ...}``)"""
        import json
        from ..utils import JSONEncoder
        if self.comm.rank == 0:
            self.logger.info('measurement done; saving result to %s' % output)
            with open(output, 'w') as ff:
                json.dump(self.__getstate__(), ff, cls=JSONEncoder)

    @classmethod
    @CurrentMPIComm.enable
    def load(cls, output, comm=None):
        """load a result written by :func:`save`"""
        import json
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


class SurveyData3PCF(SimulationBox3PCF):
    r"""
    The multipoles :math:`\zeta_\ell(r_1, r_2)` of the isotropic three-point correlation function of a survey
    catalogue, on one or several GPUs.  Runs on construction.

    The RA, Dec (degrees) and redshift columns are converted to Cartesian positions with
    :func:`~nbodykit_b200.transform.SkyToCartesian` (observer at the origin), which are then treated as
    :class:`SimulationBox3PCF` with ``periodic=False`` treats its positions: the result equals that of the
    non-periodic box on the same rows.

    Parameters
    ----------
    source : CatalogSource
        the catalogue; it provides both the primaries and the secondaries
    poles : list of int
        the multipoles to compute, distinct, from 0 up to :func:`max_ell`
    edges : array_like
        the radial bin edges in Mpc/h (see :class:`SimulationBox3PCF`)
    cosmo : Cosmology
        converts redshift into comoving distance (any object with ``comoving_distance(z)``)
    domain_factor : int, optional
        recorded in :attr:`attrs`; it has no effect (ranks take equal-width x slabs)
    ra, dec, redshift, weight : str, optional
        the column names

    Attributes
    ----------
    poles, npairs, candidates :
        as :class:`SimulationBox3PCF`
    """
    logger = logging.getLogger("SurveyData3PCF")

    def __init__(self, source, poles, edges, cosmo, domain_factor=4, ra='RA', dec='DEC', redshift='Redshift',
                 weight='Weight'):
        _verify_columns(source, None, [ra, dec, redshift, weight])
        p = _check_poles(poles)
        _check_edges(edges)
        self.source = source
        self.comm = source.comm
        self.attrs = {}
        self.attrs['poles'] = p
        self.attrs['edges'] = edges
        self.attrs['cosmo'] = cosmo
        self.attrs['periodic'] = False
        self.attrs['weight'] = weight
        self.attrs['ra'] = ra
        self.attrs['dec'] = dec
        self.attrs['redshift'] = redshift
        self.attrs['domain_factor'] = domain_factor
        self.poles = self.run()

    def _rows(self):
        from .surveypaircount import sky_rows
        a = self.attrs
        pos = sky_rows(self.source, a['ra'], a['dec'], a['redshift'], a['cosmo'], self.comm, "SurveyData3PCF")
        return pos, self._weights().to(pos.device)
