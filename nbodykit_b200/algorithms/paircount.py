"""
Pair counts and two-point correlation functions in a simulation box (API of nbodykit/algorithms/pair_counters/simbox.py
and paircount_tpcf/tpcf.py) on one or several GPUs.

The reference hands the counting to Corrfunc; here it is csrc/paircount.cu, under a contract stated in double
precision (DESIGN.md 4.6): per-axis |d| from the positions as stored (periodic: wrapped with `pos % L` in their own
dtype, then min(|d|, L - |d|)), r_p^2 = da^2 + db^2 and s^2 = r_p^2 + dc^2 with c the line of sight, bin k holding
e_k^2 <= x^2 < e_{k+1}^2.  Pairs are ordered, as Corrfunc counts them with autocorr=0: an auto count holds (i, j) and
(j, i).  Both catalogues are sorted into cells of side >= s_max / 2 with the FOF cell machinery (csrc/fof.cu).

Several GPUs: x slabs of the box (non-periodic: of the global x range).  Every pair is counted on the rank whose slab
holds its primary: rows of the first catalogue in a remote slab travel there (the slab routing with zero reach), local
ones outside the own slab are dropped, and copies of the second catalogue's rows within s_max of a remote slab travel
there.  The per-rank histograms are combined in one all-reduce.
"""
import logging
import math
import warnings

import numpy
import torch

from .. import CurrentMPIComm
from .._lib import check, darr, iarr, lib, stage
from ..binned_statistic import BinnedStatistic
from ..pmesh.pm import ParticleMesh, _ptr, _stream
from .fof import _code, _column, _sort_rows

_MODES = {'1d': 1, '2d': 2, 'projected': 3}
# the kernel modes of survey pairs, whose line of sight is the pair's midpoint as seen from the origin (DESIGN.md 4.8)
_SURVEY_KERNEL_MODES = {'1d': 1, '2d': 4, 'projected': 5, 'angular': 6}
# cells per s_max along each axis: the neighbour stencil is 5 cells wide, and the corner columns and cells whose
# nearest point is beyond s_max are skipped (DESIGN.md 4.6)
_CELLS_PER_SMAX = 2


def _second_edges(mode, Nmu, pimax):
    if mode == '2d':
        return numpy.linspace(0., 1., Nmu + 1)
    if mode == 'projected':
        return numpy.linspace(0, pimax, int(pimax + 1))
    return None


def _dims_edges(mode, edges, Nmu, pimax):
    e2 = _second_edges(mode, Nmu, pimax)
    if mode == '1d':
        return ['r'], [edges]
    if mode == '2d':
        return ['r', 'mu'], [edges, e2]
    return ['rp', 'pi'], [edges, e2]


def _smax(mode, edges, pimax):
    e = float(numpy.max(edges))
    return math.sqrt(e * e + float(pimax) ** 2) if mode == 'projected' else e


def _check_rows(n, what):
    if n >= (1 << 31):
        raise ValueError("pair count: %d rows of %s on one rank; at most 2^31 - 1 are supported" % (n, what))


class _Cells(object):
    """rows sorted into the cells of one grid: positions (double, line of sight last, wrapped when periodic), weights,
    cell table"""

    def __init__(self, pos, w, periodic, box, origin, ncell):
        n = int(pos.shape[0])
        dev = pos.device
        code = _code(pos)
        box_c, org_c, nc_c = darr(box), darr(origin), iarr(ncell)
        keys = torch.empty(n, dtype=torch.int64, device=dev)
        check(lib().nbk_fof_grid_keys(_ptr(pos), code, n, int(periodic), box_c, org_c, nc_c, _ptr(keys), _stream()),
              "nbk_fof_grid_keys")
        end_bit = max(1, (int(ncell[0]) * int(ncell[1]) * int(ncell[2]) - 1).bit_length())
        skeys, perm = _sort_rows(keys, 8, end_bit)
        del keys
        nw = int(lib().nbk_fof_compact_workspace(n))
        work = torch.empty(nw, dtype=torch.int64, device=dev)
        ncells_d = torch.empty(1, dtype=torch.int64, device=dev)
        check(lib().nbk_fof_compact_count(_ptr(skeys), n, _ptr(work), nw, _ptr(ncells_d), _stream()), "nbk_fof_compact_count")
        self.ncells = int(ncells_d.item())
        self.cell_start = torch.empty(self.ncells + 1, dtype=torch.int32, device=dev)
        self.cell_key = torch.empty(self.ncells, dtype=torch.int64, device=dev)
        check(lib().nbk_fof_compact_write(_ptr(skeys), n, _ptr(work), nw, _ptr(self.cell_start), _ptr(self.cell_key), _stream()),
              "nbk_fof_compact_write")
        del skeys, work
        spos = torch.empty_like(pos)
        check(lib().nbk_fof_sorted_pos(_ptr(pos), code, n, _ptr(perm), int(periodic), box_c, _ptr(spos), _stream()),
              "nbk_fof_sorted_pos")
        self.pos = spos.to(torch.float64).contiguous()           # exact: f4 -> f8 after the wrap in f4
        self.w = w.index_select(0, perm.to(torch.int64)).contiguous()
        self.n = n

    def chunks(self, rows):
        """(chunk_first[nchunks + 1], chunk_key[nchunks]): every cell split into runs of at most `rows` rows"""
        dev = self.cell_start.device
        cs = self.cell_start.to(torch.int64)
        nch = (cs[1:] - cs[:-1] + (rows - 1)) // rows
        first_chunk = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), torch.cumsum(nch, 0)])
        nchunks = int(first_chunk[-1].item())
        cell = torch.repeat_interleave(torch.arange(self.ncells, dtype=torch.int64, device=dev), nch)
        first = cs[cell] + (torch.arange(nchunks, dtype=torch.int64, device=dev) - first_chunk[cell]) * rows
        first = torch.cat([first, torch.full((1,), self.n, dtype=torch.int64, device=dev)])
        return first.contiguous(), self.cell_key[cell].contiguous(), nchunks


def count_pairs(mode, pos1, w1, pos2, w2, edges, periodic, box, los=2, Nmu=None, pimax=None, survey=False):
    """binned ordered pairs of the rows of pos1 (primaries) against those of pos2 on this device, per the contract of
    DESIGN.md 4.6 (``survey``: of 4.8, not periodic, with the observer at the origin; 'angular' takes unit vectors and
    chord edges).  pos: (n, 3) float32 / float64 device tensors in box coordinates; w: float64 (n,).  Returns device
    tensors (npairs int64, wsum f64, sepsum f64) of nbins entries and the number of candidate pairs tested."""
    dev = pos1.device
    axes = [i for i in range(3) if i != los] + [los]
    e1 = numpy.asarray(edges, dtype='f8')
    e2 = _second_edges(mode, Nmu, pimax)
    nbins = (len(e1) - 1) * (1 if e2 is None else len(e2) - 1)
    npairs = torch.zeros(nbins, dtype=torch.int64, device=dev)
    wsum = torch.zeros(nbins, dtype=torch.float64, device=dev)
    ssum = torch.zeros(nbins, dtype=torch.float64, device=dev)
    cand = torch.zeros(1, dtype=torch.int64, device=dev)
    n1, n2 = int(pos1.shape[0]), int(pos2.shape[0])
    if n1 == 0 or n2 == 0:
        return npairs, wsum, ssum, 0
    p1 = pos1[:, axes].contiguous()
    p2 = pos2[:, axes].contiguous()
    if periodic:
        gbox = numpy.asarray(box, 'f8')[axes]
        origin = numpy.zeros(3)
    else:
        lo = torch.minimum(p1.min(0).values.double(), p2.min(0).values.double()).cpu().numpy()
        hi = torch.maximum(p1.max(0).values.double(), p2.max(0).values.double()).cpu().numpy()
        origin = lo
        gbox = numpy.where(hi > lo, hi - lo, 1.0)
    smax = _smax(mode, e1, pimax)
    ncell = [int(min(max(1, math.floor(L * _CELLS_PER_SMAX / (smax * (1 + 1e-4)))), 1 << 20)) for L in gbox]
    # a row may sit outside its cell by the rounding of its cell index, or by L_f4 - L_f8 when an f4 position wraps to L
    tol = 4e-7 * (gbox + numpy.abs(origin))
    with stage("paircount_cells"):
        c2 = _Cells(p2, w2, periodic, gbox, origin, ncell)
        del p2
        c1 = _Cells(p1, w1, periodic, gbox, origin, ncell)
        del p1
        first, ckey, nchunks = c1.chunks(int(lib().nbk_paircount_chunk_rows()))
    work = torch.empty(len(e1) + (2 if e2 is None else len(e2)), dtype=torch.float64, device=dev)
    kmode = (_SURVEY_KERNEL_MODES if survey else _MODES)[mode]
    with stage("paircount_count"):
        check(lib().nbk_paircount(kmode, _ptr(c1.pos), _ptr(c1.w), _ptr(first), _ptr(ckey), nchunks, _ptr(c2.pos), _ptr(c2.w),
                                  _ptr(c2.cell_start), _ptr(c2.cell_key), c2.ncells, int(periodic), darr(gbox), iarr(ncell),
                                  darr(tol), darr(e1), len(e1), darr(e2) if e2 is not None else None,
                                  len(e2) if e2 is not None else 0, float(pimax or 0.0), _ptr(work), _ptr(npairs), _ptr(wsum),
                                  _ptr(ssum), _ptr(cand), _stream()), "nbk_paircount")
    return npairs, wsum, ssum, int(cand.item())


def slab_route(comm, pos1, w1, pos2, w2, periodic, box, smax):
    """(primaries, their weights, secondaries, their weights) of this rank's x slab: every row of pos1 on the rank
    whose slab holds it, and every row of pos2 on its own rank plus copies on each remote slab within smax of it"""
    P = comm.size
    if periodic:
        rbox = box
        r1, r2 = pos1, pos2
    else:
        def bounds(p):
            if p.shape[0] == 0:
                return numpy.inf, -numpy.inf
            x = p[:, 0]
            return float(x.min().item()), float(x.max().item())
        b = [bounds(pos1), bounds(pos2)]
        lo = min(min(v[0] for v in comm.allgather(bb)) for bb in b)
        hi = max(max(v[1] for v in comm.allgather(bb)) for bb in b)
        lo = lo if numpy.isfinite(lo) else 0.0
        rbox = numpy.array([hi - lo if hi > lo else 1.0, 1.0, 1.0])
        # slabs of [lo, hi] in double, so that the shift by lo cannot move a row across a slab edge
        r1 = pos1.to(torch.float64, copy=True)
        r1[:, 0] -= lo
        r2 = r1 if pos2 is pos1 else pos2.to(torch.float64, copy=True)
        if pos2 is not pos1:
            r2[:, 0] -= lo
    pm = ParticleMesh(BoxSize=rbox, Nmesh=[P, P, P], dtype='f8', comm=comm)
    # primaries: every row belongs to the one slab holding floor(x P / Lx); rows listed by the zero-reach routing
    # are remote, all others stay
    lay1 = pm._decompose_device(r1, 0.0)
    keep = torch.ones(int(pos1.shape[0]), dtype=torch.bool, device=pos1.device)
    if lay1.ghosts.numel():
        keep[(lay1.ghosts & 0xffffffff)] = False
    rp1, rw1 = lay1.route(pos1, mass=w1)
    prim = torch.cat([pos1[keep], rp1])
    pw = torch.cat([w1[keep], rw1])
    # secondaries: copies of the rows within s_max of a remote slab, widened a little so that the rounding of
    # x P / Lx can never drop a needed copy; a reach of P + 1 slabs already reaches every slab
    smoothing = min(smax * P / float(rbox[0]) * (1 + 1e-6) + 1e-9, P + 1.0)
    lay2 = pm._decompose_device(r2, smoothing)
    rp2, rw2 = lay2.route(pos2, mass=w2)
    sec = torch.cat([pos2, rp2])
    sw = torch.cat([w2, rw2])
    return prim.contiguous(), pw.contiguous(), sec.contiguous(), sw.contiguous()


def reduce_histograms(comm, npairs, wsum, ssum, cand):
    """host arrays of the count_pairs histograms summed over ranks, in one all-reduce (counts as two exact 32-bit
    halves)"""
    if comm.size == 1:
        return npairs.cpu().numpy().astype('u8'), wsum.cpu().numpy(), ssum.cpu().numpy(), int(cand)
    c = torch.cat([npairs, torch.tensor([cand], dtype=torch.int64, device=npairs.device)])
    packed = torch.cat([(c & 0xffffffff).to(torch.float64), (c >> 32).to(torch.float64), wsum, ssum])
    comm.allreduce_tensor(packed, "sum")
    k = c.shape[0]
    lo = packed[:k].round().to(torch.int64)
    hi = packed[k:2 * k].round().to(torch.int64)
    tot = (hi << 32) + lo
    nb = npairs.shape[0]
    return (tot[:nb].cpu().numpy().astype('u8'), packed[2 * k:2 * k + nb].cpu().numpy(),
            packed[2 * k + nb:].cpu().numpy(), int(tot[nb].item()))


def _verify_columns(first, second, columns):
    """both sources (second None: the first) share a communicator and hold `columns`"""
    if second is None:
        second = first
    assert second.comm is first.comm, "communicator mismatch between input sources"
    for source in (first, second):
        for col in columns:
            if col not in source:
                raise ValueError("the column '%s' is missing from input source; cannot do pair count" % col)


def weight_column(source, name):
    """a source's weight column as a contiguous float64 (n,) tensor on the GPU"""
    col = source[name]
    if hasattr(col, 'materialize'):
        col = col.materialize()
    col = col.compute() if hasattr(col, 'compute') else col
    t = torch.as_tensor(col)
    if not t.is_cuda:
        t = t.cuda()
    return t.to(torch.float64).reshape(-1).contiguous()


def _verify_sources(first, second, BoxSize, columns):
    """the box of the count from the sources' attrs and the `BoxSize` keyword; every source must hold `columns`"""
    _verify_columns(first, second, columns)
    if second is None:
        second = first
    box = numpy.zeros(3)
    b1 = first.attrs.get('BoxSize', None)
    b2 = second.attrs.get('BoxSize', None)
    if b1 is not None:
        box[:] = b1
    if BoxSize is not None:
        box[:] = BoxSize
    if (box == 0.).all():
        raise ValueError("BoxSize must be supplied in the source ``attrs`` or via the ``BoxSize`` keyword")
    if b1 is not None and b2 is not None:
        if not numpy.all(numpy.asarray(b1) == numpy.asarray(b2)):
            raise ValueError("BoxSize mismatch between pair count cross-correlation sources")
        if not numpy.all(numpy.asarray(b1) == box):
            raise ValueError("BoxSize mismatch between sources and the pair count algorithm")
    return box


def check_pair_args(mode, edges, Nmu, pimax):
    """the argument checks of the reference's PairCountBase, and those of the bin edges (as float64, returned)"""
    if mode not in ['1d', '2d', 'projected', 'angular']:
        raise ValueError("allowed 'mode' values are: %s" % ['1d', '2d', 'projected', 'angular'])
    if numpy.min(edges) <= 0.:
        raise ValueError("the lower edge of the 1st separation bin must greater than zero (no self-pairs)")
    if mode == '2d' and Nmu is None:
        raise ValueError("'Nmu' keyword is required when 'mode' is '2d'")
    if Nmu is not None and mode != '2d':
        raise ValueError("mode should be '2d' if 'Nmu' is specified")
    if mode == 'projected' and pimax is None:
        raise ValueError("'pimax' keyword is required when 'mode' is 'projected'")
    if pimax is not None and mode != 'projected':
        raise ValueError("mode should be 'projected' if 'projected' is specified")
    if mode == 'projected' and pimax < 1.0:
        raise ValueError("'pimax' must be at least 1.0 when 'mode' is 'projected'")
    e = numpy.asarray(edges, dtype='f8')
    if e.ndim != 1 or len(e) < 2 or not numpy.isfinite(e).all() or not (numpy.diff(e) > 0).all():
        raise ValueError("pair count: edges must be a 1-D array of at least two finite, strictly increasing values")
    if mode == '2d' and (int(Nmu) != Nmu or Nmu < 1):
        raise ValueError("pair count: Nmu must be a positive integer")
    return e


class BasePairCount(object):
    """a pair-count result (``pairs``, ``attrs``), saved and loaded as JSON; subclasses rebuild ``pairs`` in
    ``__setstate__``"""

    def __getstate__(self):
        return {'pairs': self.pairs.data, 'attrs': self.attrs}

    def save(self, output):
        """save the result as JSON (``{'pairs': ..., 'attrs': ...}``)"""
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


class SimulationBoxPairCount(BasePairCount):
    r"""
    Count (weighted) pairs of objects in a simulation box as a function of :math:`r`, :math:`(r, \mu)` or
    :math:`(r_p, \pi)`, on one or several GPUs.  Runs on construction.

    Parameters
    ----------
    mode : '1d', '2d', 'projected'
        bin in the separation, in (separation, mu) or in (r_p, pi); 'angular' raises NotImplementedError
    first : CatalogSource
        the primary catalogue
    edges : array_like
        the separation (or r_p) bin edges, positive, finite and strictly increasing
    BoxSize : float, 3-vector, optional
        the box; if not given, ``first.attrs['BoxSize']``
    periodic : bool, optional
        minimum-image separations in a cubic box
    second : CatalogSource, optional
        the catalogue to cross-correlate with; None (or ``first``) counts the auto pairs
    los : 'x', 'y', 'z' or 0, 1, 2
        the line-of-sight axis
    Nmu : int, optional
        mu bins over [0, 1] ('2d' only)
    pimax : float, optional
        the largest line-of-sight separation ('projected' only); pi bins are ``linspace(0, pimax, int(pimax + 1))``
    weight : str, optional
        the weight column; each pair counts ``w_i * w_j`` in ``wnpairs``
    position : str, optional
        the position column
    show_progress : bool, optional
        recorded in :attr:`attrs`; it has no effect (there is no Corrfunc chunk loop to report on)
    **config :
        recorded in :attr:`attrs`; they have no effect, because no Corrfunc call takes them

    Pairs are ordered, as Corrfunc counts them: an auto count holds (i, j) and (j, i).  At most 2^31 - 1 rows of each
    catalogue per rank.

    Attributes
    ----------
    pairs : BinnedStatistic
        dims ``['r']``, ``['r', 'mu']`` or ``['rp', 'pi']``; variables ``r`` / ``rp`` (unweighted mean separation of
        the pairs in the bin, 0 when empty), ``npairs`` (u8) and ``wnpairs`` (sum of w_i * w_j)
    """
    logger = logging.getLogger('SimulationBoxPairCount')

    def __init__(self, mode, first, edges, BoxSize=None, periodic=True, second=None, los='z', Nmu=None, pimax=None,
                 weight='Weight', position='Position', show_progress=False, **config):
        if isinstance(los, str):
            if los not in 'xyz' or len(los) != 1:
                raise ValueError("``los`` should be one of 'x', 'y', 'z'")
            los = 'xyz'.index(los)
        if isinstance(los, (int, numpy.integer)) and los < 0:
            los += 3
        if los not in [0, 1, 2]:
            raise ValueError("``los`` should be either ['x', 'y', 'z'] or [0,1,2]")
        los = int(los)

        BoxSize = _verify_sources(first, second, BoxSize, [position, weight])

        check_pair_args(mode, edges, Nmu, pimax)
        if mode == 'angular':
            raise NotImplementedError("mode='angular' needs the Cartesian to RA/Dec transform (CartesianToEquatorial) "
                                      "and an angular pair counter, which nbodykit_b200 does not have")

        self.first = first
        self.second = second
        self.comm = first.comm
        self.attrs = {}
        self.attrs['mode'] = mode
        self.attrs['edges'] = edges
        self.attrs['Nmu'] = Nmu
        self.attrs['pimax'] = pimax
        self.attrs['show_progress'] = show_progress
        self.attrs['N1'] = first.csize
        self.attrs['N2'] = second.csize if second is not None else None
        self.attrs['BoxSize'] = BoxSize
        self.attrs['periodic'] = periodic
        self.attrs['weight'] = weight
        self.attrs['position'] = position
        self.attrs['config'] = config
        self.attrs['los'] = los

        if periodic:
            half = 0.5 * BoxSize.min()
            if numpy.amax(edges) > half or (mode == 'projected' and pimax > half):
                raise ValueError("periodic pair counts cannot be computed for Rmax > BoxSize/2")
            if not numpy.all(BoxSize == BoxSize[0]):
                raise NotImplementedError("periodic wrapping with non-cubic boxes not implemented yet")
        self.run()

    def _weights(self, source):
        return weight_column(source, self.attrs['weight'])

    def run(self):
        """count the pairs; sets :attr:`pairs` and ``attrs['total_wnpairs']`` / ``attrs['is_cross']``"""
        comm = self.comm
        attrs = self.attrs
        mode, periodic = attrs['mode'], bool(attrs['periodic'])
        first, second = self.first, self.second
        auto = second is None or second is first
        pos1 = _column(first, attrs['position'], None)
        if pos1.ndim != 2 or pos1.shape[1] != 3:
            raise ValueError("pair count: Position must have shape (n, 3)")
        w1 = self._weights(first)
        if auto:
            pos2, w2 = pos1, w1
        else:
            pos2 = _column(second, attrs['position'], pos1.device)
            w2 = self._weights(second)
        _check_rows(int(pos1.shape[0]), "the first catalogue")
        _check_rows(int(pos2.shape[0]), "the second catalogue")

        # the normalisation of the estimators (0.5 by convention; it cancels in every ratio)
        s1 = comm.allreduce(float(w1.sum().item()))
        if auto:
            s2 = comm.allreduce(float((w1 * w1).sum().item()))
            attrs['total_wnpairs'] = 0.5 * (s1 ** 2 - s2)
            attrs['is_cross'] = False
        else:
            s2 = comm.allreduce(float(w2.sum().item()))
            attrs['total_wnpairs'] = 0.5 * s1 * s2
            attrs['is_cross'] = True

        box = numpy.asarray(attrs['BoxSize'], 'f8')
        smax = _smax(mode, attrs['edges'], attrs['pimax'])
        with stage("paircount_route"):
            if comm.size > 1:
                pos1, w1, pos2, w2 = self._route(pos1, w1, pos2, w2, periodic, box, smax)
                _check_rows(int(pos1.shape[0]), "primaries after routing")
                _check_rows(int(pos2.shape[0]), "secondaries after routing")
        npairs, wsum, ssum, cand = count_pairs(mode, pos1, w1, pos2, w2, attrs['edges'], periodic, box, attrs['los'],
                                               attrs['Nmu'], attrs['pimax'])
        with stage("paircount_reduce"):
            npairs, wsum, ssum, cand = self._reduce(npairs, wsum, ssum, cand)
        self.candidates = cand

        dims, edges = _dims_edges(mode, attrs['edges'], attrs['Nmu'], attrs['pimax'])
        shape = tuple(len(e) - 1 for e in edges)
        data = numpy.zeros(shape, dtype=[(dims[0], 'f8'), ('npairs', 'u8'), ('wnpairs', 'f8')])
        n = npairs.reshape(shape)
        data['npairs'] = n
        data['wnpairs'] = wsum.reshape(shape)
        sep = numpy.zeros(shape)
        numpy.divide(ssum.reshape(shape), n, out=sep, where=n > 0)
        data[dims[0]] = sep
        self.pairs = BinnedStatistic(dims, edges, data, fields_to_sum=['npairs', 'wnpairs'])
        self.pairs.attrs['total_wnpairs'] = attrs['total_wnpairs']

    def _route(self, pos1, w1, pos2, w2, periodic, box, smax):
        """(primaries, their weights, secondaries, their weights) of this rank's x slab"""
        return slab_route(self.comm, pos1, w1, pos2, w2, periodic, box, smax)

    def _reduce(self, npairs, wsum, ssum, cand):
        """host arrays of the histograms summed over ranks, in one all-reduce (counts as two exact 32-bit halves)"""
        return reduce_histograms(self.comm, npairs, wsum, ssum, cand)

    # ------------------------------------------------------------------------------------------------------------------
    def __setstate__(self, state):
        self.__dict__.update(state)
        a = self.attrs
        if a['mode'] not in _MODES:
            raise ValueError("mode = '%s' should be one of %s" % (a['mode'], list(_MODES)))
        dims, edges = _dims_edges(a['mode'], a['edges'], a['Nmu'], a['pimax'])
        self.pairs = BinnedStatistic(dims, edges, self.pairs, fields_to_sum=['npairs', 'wnpairs'])


# ---- estimators ------------------------------------------------------------------------------------------------------
class WedgeBinnedStatistic(BinnedStatistic):
    """a BinnedStatistic of mu wedges that converts to multipoles"""

    def to_poles(self, poles):
        r"""
        the multipoles :math:`\xi_\ell(r)` of the wedges :math:`\xi(r, \mu)`: the sum over the mu bins of
        :math:`(2\ell + 1) L_\ell(\mu_c)\, \xi\, \Delta\mu` over the summed :math:`\Delta\mu`, with :math:`\mu_c` the
        centre of each mu bin.  Select a mu range first with ``self.sel(mu=slice(lo, hi), method='nearest')``.
        """
        from scipy.special import eval_legendre
        x = str(self.dims[0])
        mu = self.edges['mu']
        dmu = numpy.diff(mu)
        centre = 0.5 * (mu[1:] + mu[:-1])
        data = numpy.zeros(self.shape[0], dtype=[(x, 'f8')] + [('corr_%d' % ell, 'f8') for ell in poles])
        for ell in poles:
            kernel = (2. * ell + 1.) * eval_legendre(ell, centre)
            data['corr_%d' % ell] = (self['corr'] * kernel * dmu).sum(axis=-1) / dmu.sum()
        data[x] = numpy.mean(self[x], axis=-1)
        return BinnedStatistic(dims=[x], edges=[self.edges[x]], data=data, poles=poles)


def filling_factor(mode, edges, BoxSize):
    """the fraction of the box volume in each bin, for the analytic uniform randoms: spherical shells ('1d'), shells
    cut into |mu| sectors ('2d', both hemispheres) or cylindrical annuli of height 2 pi ('projected'); `edges` is the
    dict of bin edges by dimension"""
    V = numpy.prod(numpy.asarray(BoxSize, 'f8'))
    if mode == '1d':
        r = numpy.asarray(edges['r'], 'f8')
        return numpy.diff(4. * numpy.pi / 3. * r ** 3) / V
    if mode == '2d':
        r, mu = numpy.asarray(edges['r'], 'f8'), numpy.asarray(edges['mu'], 'f8')
        shell = numpy.diff(4. * numpy.pi / 3. * r ** 3)           # the full shell, both signs of mu
        return numpy.outer(shell, numpy.diff(mu)) / V
    if mode == 'projected':
        rp, pi = numpy.asarray(edges['rp'], 'f8'), numpy.asarray(edges['pi'], 'f8')
        return numpy.outer(numpy.diff(numpy.pi * rp ** 2), numpy.diff(2. * pi)) / V
    raise ValueError("no analytic randoms for mode '%s'" % mode)


class _AnalyticPairs(object):
    """the expected pair counts of uniform randoms, shaped like a pair count (``.pairs``, ``.attrs``)"""

    def __init__(self, mode, dims, edges, BoxSize, N1, N2=None):
        f = filling_factor(mode, edges, BoxSize)
        if N2 is None:
            rr, total = N1 * N1 * f, 0.5 * N1 * (N1 - 1.)
        else:
            rr, total = N1 * N2 * f, 0.5 * N1 * N2
        data = numpy.zeros(rr.shape, dtype=[('npairs', 'f8'), ('wnpairs', 'f8')])
        data['npairs'] = rr
        data['wnpairs'] = rr
        self.pairs = WedgeBinnedStatistic(dims, [edges[d] for d in dims], data)
        self.attrs = {'total_wnpairs': total}
        self.pairs.attrs['total_wnpairs'] = total


def _tpcf_result(D1D2, corr):
    x = D1D2.dims[0]
    data = numpy.zeros(corr.shape, dtype=[('corr', 'f8'), (x, 'f8')])
    data['corr'] = corr
    data[x] = D1D2[x]
    return WedgeBinnedStatistic(D1D2.dims, [D1D2.edges[d] for d in D1D2.dims], data)


def natural_estimator(D1D2):
    """(R1R2 pairs, corr): DD / RR - 1 against analytic uniform randoms, both normalised by their total_wnpairs"""
    a = D1D2.attrs
    N2 = a['N2'] if a['is_cross'] else None
    R = _AnalyticPairs(a['mode'], D1D2.pairs.dims, D1D2.pairs.edges, a['BoxSize'], a['N1'], N2)
    scale = R.attrs['total_wnpairs'] / a['total_wnpairs']
    corr = D1D2.pairs['wnpairs'] * scale / R.pairs['wnpairs'] - 1.
    return R.pairs, _tpcf_result(D1D2.pairs, corr)


def landy_szalay(D1D2, D1R2, D2R1, R1R2):
    """corr = (f_DD DD - f_DR DR - f_RD RD) / RR + 1, each term normalised to R1R2's total_wnpairs; NaN where RR
    holds no pairs"""
    tot = R1R2.attrs['total_wnpairs']
    RR = R1R2.pairs['wnpairs']
    ok = R1R2.pairs['npairs'] > 0
    corr = numpy.full(D1D2.pairs.shape, numpy.nan)
    num = (tot / D1D2.attrs['total_wnpairs']) * D1D2.pairs['wnpairs'] \
        - (tot / D1R2.attrs['total_wnpairs']) * D1R2.pairs['wnpairs'] \
        - (tot / D2R1.attrs['total_wnpairs']) * D2R1.pairs['wnpairs']
    corr[ok] = num[ok] / RR[ok] + 1.
    if not ok.all():
        warnings.warn("Landy-Szalay: some separation bins hold no random pairs; their correlation is NaN. Use more "
                      "randoms or broader bins.")
    return _tpcf_result(D1D2.pairs, corr)


def projected_wp(corr):
    r"""w_p(r_p) = 2 \sum_\pi \xi(r_p, \pi) \Delta\pi"""
    wp = 2. * (corr['corr'] * numpy.diff(corr.edges['pi'])).sum(axis=-1)
    out = corr.copy().average('pi')
    out['corr'] = wp
    return out


def _wedge(b):
    return b if b is None or isinstance(b, WedgeBinnedStatistic) else b.copy(cls=WedgeBinnedStatistic)


class BasePairCount2PCF(object):
    """the result of a pair-count correlation function: ``corr``, the pair counts ``D1D2``, ``D1R2``, ``D2R1``,
    ``R1R2`` and ``wp`` (WedgeBinnedStatistic or None), ``attrs``; saved and loaded as JSON"""

    def __getstate__(self):
        state = {'corr': self.corr.data, 'dims': self.corr.dims, 'edges': [self.corr.edges[d] for d in self.corr.dims]}
        for name in ('D1D2', 'D1R2', 'D2R1', 'R1R2', 'wp'):
            v = getattr(self, name, None)
            state[name] = v.data if v is not None else None
        state['attrs'] = self.attrs
        return state

    def __setstate__(self, state):
        state = dict(state)
        edges, dims = state.pop('edges'), state.pop('dims')
        self.__dict__.update(state)
        self.corr = WedgeBinnedStatistic(dims, edges, self.corr)
        if self.wp is not None:
            self.wp = WedgeBinnedStatistic(dims[:1], edges[:1], self.wp)
        for name in ('D1D2', 'D1R2', 'D2R1', 'R1R2'):
            v = getattr(self, name)
            if v is not None:
                setattr(self, name, WedgeBinnedStatistic(dims, edges, v))

    def save(self, output):
        """save the result as JSON"""
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


class SimulationBox2PCF(BasePairCount2PCF):
    r"""
    The two-point correlation function of catalogues in a simulation box, from pair counts, as a function of
    :math:`r`, :math:`(r, \mu)` or :math:`(r_p, \pi)`.  Runs on construction.

    Periodic with no ``randoms1``: the natural estimator DD / RR - 1 against analytic uniform randoms (assumed
    unweighted).  Otherwise the Landy-Szalay estimator over the catalogue randoms (``randoms2`` defaults to
    ``randoms1``); a given ``R1R2`` (a :class:`SimulationBoxPairCount`) is used instead of counting the random pairs.
    The other parameters are those of :class:`SimulationBoxPairCount`; ``show_progress`` and ``**config`` are recorded
    and have no effect.

    Attributes
    ----------
    D1D2, D1R2, D2R1, R1R2 : WedgeBinnedStatistic
        the pair counts (D1R2 / D2R1 are None with analytic randoms)
    corr : WedgeBinnedStatistic
        the correlation function (``corr``) and the mean separation of the D1D2 pairs
    wp : WedgeBinnedStatistic
        ``'projected'`` only: :math:`w_p(r_p) = 2 \sum \xi \Delta\pi` in ``corr``
    """
    logger = logging.getLogger('SimulationBox2PCF')

    def __init__(self, mode, data1, edges, Nmu=None, pimax=None, data2=None, randoms1=None, randoms2=None, R1R2=None,
                 periodic=True, BoxSize=None, los='z', weight='Weight', position='Position', show_progress=False, **config):
        self.comm = data1.comm
        self.attrs = {'mode': mode, 'edges': numpy.array(edges), 'Nmu': Nmu, 'pimax': pimax, 'periodic': periodic,
                      'BoxSize': BoxSize, 'los': los, 'weight': weight, 'position': position,
                      'show_progress': show_progress, 'config': config}
        self.data1, self.data2 = data1, data2
        self.randoms1, self.randoms2 = randoms1, randoms2
        self.R1R2 = R1R2
        self.run()

    def run(self):
        """count the pairs and apply the estimator; sets D1D2, D1R2, D2R1, R1R2, corr (and wp)"""
        kw = dict(self.attrs)
        kw.update(kw.pop('config'))
        if kw['periodic'] and self.randoms1 is None:
            DD = SimulationBoxPairCount(first=self.data1, second=self.data2, **kw)
            RR, self.corr = natural_estimator(DD)
            self.D1D2, self.R1R2 = DD.pairs, RR
            self.D1R2 = self.D2R1 = None
        else:
            if self.randoms1 is None:
                raise ValueError("a catalog of randoms must be specified as the ``randoms1`` keyword when the data is "
                                 "not in a simulation box with periodic boundary conditions")
            if self.data2 is not None and self.randoms2 is None:
                self.randoms2 = self.randoms1
            r2 = self.randoms2 if self.randoms2 is not None else self.randoms1
            RR = self.R1R2
            if RR is None:
                RR = SimulationBoxPairCount(first=self.randoms1, second=r2, **kw)
            DD = SimulationBoxPairCount(first=self.data1, second=self.data2, **kw)
            DR = SimulationBoxPairCount(first=self.data1, second=r2, **kw)
            RD = SimulationBoxPairCount(first=self.data2, second=self.randoms1, **kw) if self.data2 is not None else DR
            self.corr = landy_szalay(DD, DR, RD, RR)
            self.D1D2, self.D1R2, self.D2R1, self.R1R2 = DD.pairs, DR.pairs, RD.pairs, RR.pairs
        for name in ('D1D2', 'D1R2', 'D2R1', 'R1R2'):
            setattr(self, name, _wedge(getattr(self, name)))
        self.wp = projected_wp(self.corr) if self.attrs['mode'] == 'projected' else None
