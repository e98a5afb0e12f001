"""
Nearest-neighbour density estimate (API of nbodykit/algorithms/kdtree.py: KDDensity) on one or several GPUs.

Contract (DESIGN.md 4.10).  q = pos / L in the positions' own dtype (float32: f4(f8(x) / L)), then numpy's q % 1 in
that dtype; a q that rounds to 1.0 becomes 0.0.  d is the 8th smallest distance from a row to all rows of the catalogue,
itself included: per axis dx = q_a - q_b in double, dx > 0.5 -> dx - 1, dx < -0.5 -> dx + 1, d = sqrt((dx^2 + dy^2) +
dz^2).  density = 1 / (d^3 V).  With 8 or more coincident rows d = 0 (density inf); with fewer than 8 rows in all d = inf
(density 0).  This is the reference's answer on one rank, and it does not depend on the number of ranks or on `margin`.

The kernels (csrc/kdtree.cu) keep a sorted list of the 8 smallest squared distances per query in registers and walk
Chebyshev rings of cells of the unit box around it until the next ring cannot beat the 8th.

Several GPUs: x slabs of the unit box.  Phase 1: every row moves to the slab that holds it, copies of the rows within
h = margin (1 / N)^(1/3) of a remote slab travel there, and every owned row finds its 8th distance among the owned rows
and the copies.  It is exact when it is no larger than the row's x-distance to the outer edge of the copies.  Phase 2:
every other row travels as a query to each remote slab within its phase-1 distance, every rank returns the 8 smallest
distances to its owned rows, and the owner takes the 8th smallest of them all.
"""
import logging
import math

import numpy
import torch

from .._lib import check, iarr, lib, stage
from ..pmesh.pm import ParticleMesh, _ptr, _stream
from .fof import _column
from .paircount import _Cells

# rows per cell at the mean density of the whole catalogue (DESIGN.md 4.10)
_ROWS_PER_CELL = 4.0
# the dense cell table holds 4 bytes per cell of the whole grid on every rank
_MAX_CELLS_PER_AXIS = 1024


class KDDensity(object):
    """
    Estimate a proxy density based on the distance to the nearest neighbours: the inverse cube of the distance to the
    8th nearest row, the row itself included, times the box volume.  Runs on construction; the result is
    :attr:`density`.

    Parameters
    ----------
    source : CatalogSource
        the input source of particles; must have a 'Position' column and a cubic 'BoxSize' attribute
    margin : float, optional
        the width of the slab halo of the first pass on several ranks, in units of the mean separation
        ``(V / csize)^(1/3)``.  It changes the speed only, never the result

    Divergences from the reference:

    - a unit coordinate that rounds to 1.0 (float32 positions just below 0) becomes 0.0; the reference's cKDTree raises
      ``ValueError`` there;
    - on several ranks the result is the one-rank answer for every row; the reference's halo of
      ``margin * attrs['meansep']`` is too thin to find the neighbours of rows near its domain faces;
    - a non-cubic box raises ``ValueError``, where the reference asserts.

    At most 2^31 - 1 rows per rank, copies included.

    Attributes
    ----------
    density : numpy.ndarray
        float64, one value per local row, in the source's order
    attrs : dict
        ``BoxSize`` (float64 3-vector), ``meansep`` and ``margin``.  ``meansep`` keeps the reference's value,
        ``(csize / V)^(1/3)``: the cube root of the number density, not the mean separation
    """
    logger = logging.getLogger('KDDensity')

    def __init__(self, source, margin=1.0):
        if 'Position' not in source:
            raise ValueError("please specify the 'Position' column in the input source")

        self.comm = source.comm
        self._source = source

        if 'BoxSize' not in source.attrs:
            raise ValueError("please specify 'BoxSize' in the input source 'attrs'")
        BoxSize = numpy.array(source.attrs['BoxSize'], dtype='f8')
        if BoxSize.ndim == 0 or BoxSize.size == 1:
            BoxSize = numpy.repeat(BoxSize.reshape(-1), 3)
        if BoxSize.shape != (3,):
            raise ValueError("KDDensity: BoxSize must be a scalar or a 3-vector (got shape %s)" % str(BoxSize.shape))
        if not numpy.all(BoxSize == BoxSize[0]):
            raise ValueError("KDDensity needs a cubic box (got BoxSize %s)" % str(BoxSize))
        if not (numpy.isfinite(BoxSize[0]) and BoxSize[0] > 0):
            raise ValueError("KDDensity: BoxSize must be positive and finite (got %s)" % str(BoxSize))
        if not (numpy.isscalar(margin) and numpy.isfinite(float(margin)) and float(margin) >= 0):
            raise ValueError("KDDensity: ``margin`` must be a non-negative finite number (got %r)" % (margin,))
        if source.size >= (1 << 31):
            raise ValueError("KDDensity: %d rows on one rank; at most 2^31 - 1 are supported" % source.size)

        self.attrs = {}
        self.attrs['BoxSize'] = BoxSize
        self.attrs['meansep'] = (source.csize / BoxSize.prod()) ** (1.0 / len(BoxSize))
        self.attrs['margin'] = margin

        self.run()

    def run(self):
        """compute :attr:`density` (and the distances, in ``_distance``)"""
        comm = self.comm
        L = float(self.attrs['BoxSize'][0])
        pos = _column(self._source, 'Position', None)
        if pos.ndim != 2 or pos.shape[1] != 3:
            raise ValueError("KDDensity: Position must have shape (n, 3)")
        n = int(pos.shape[0])
        with stage("kd_unit"):
            q = unit_positions(pos, L)
            del pos
        N = int(self._source.csize)
        d2, self._stats = kth_distance2(comm, q, N, float(self.attrs['margin']))
        with stage("kd_density"):
            dist = torch.empty(n, dtype=torch.float64, device=q.device)
            dens = torch.empty(n, dtype=torch.float64, device=q.device)
            check(lib().nbk_kd_density(_ptr(d2), n, float(self.attrs['BoxSize'].prod()), _ptr(dist), _ptr(dens), _stream()),
                  "nbk_kd_density")
        self._distance = dist.cpu().numpy()
        self.density = dens.cpu().numpy()


def unit_positions(pos, L):
    """the unit coordinates q of device positions (n, 3) in a box of side L, as double"""
    n = int(pos.shape[0])
    q = torch.empty((n, 3), dtype=torch.float64, device=pos.device)
    code = 4 if pos.dtype == torch.float32 else 8
    check(lib().nbk_kd_unit(_ptr(pos), code, n, float(L), _ptr(q), _stream()), "nbk_kd_unit")
    return q


def _ncell(N):
    """cells per axis of the unit box: about _ROWS_PER_CELL rows per cell at the mean density of N rows"""
    c = int(math.floor((max(N, 1) / _ROWS_PER_CELL) ** (1 / 3.) * (1 + 1e-12)))
    return [min(max(1, c), _MAX_CELLS_PER_AXIS)] * 3


class _Grid(object):
    """the rows q (owned first, then copies) sorted into the cells of the unit box, with a dense cell table"""

    def __init__(self, q, n_own, ncell):
        n = int(q.shape[0])
        dev = q.device
        self.n, self.n_own, self.ncell = n, n_own, ncell
        self.nc_c = iarr(ncell)
        cells = _Cells(q, torch.zeros(n, dtype=torch.uint8, device=dev), True, numpy.ones(3), numpy.zeros(3), ncell)
        self.pos = cells.pos
        self.perm = cells.perm
        ntot = ncell[0] * ncell[1] * ncell[2]
        self.dense = torch.empty(ntot + 1, dtype=torch.int32, device=dev)
        check(lib().nbk_kd_cell_table(_ptr(cells.cell_start), _ptr(cells.cell_key), cells.ncells, self.nc_c, _ptr(self.dense),
                                      _stream()), "nbk_kd_cell_table")

    def self_kth(self, cand):
        """the 8th smallest d2 of every owned row (row order) to all rows"""
        kth = torch.empty(self.n_own, dtype=torch.float64, device=self.pos.device)
        check(lib().nbk_kd_self(_ptr(self.pos), _ptr(self.perm), self.n, self.n_own, _ptr(self.dense), self.nc_c, _ptr(kth),
                                _ptr(cand), _stream()), "nbk_kd_self")
        return kth

    def query(self, qpos, cand):
        """the 8 smallest d2, ascending, from every row of qpos to the owned rows"""
        K = int(lib().nbk_kd_k())
        nq = int(qpos.shape[0])
        knn = torch.empty((nq, K), dtype=torch.float64, device=qpos.device)
        check(lib().nbk_kd_query(_ptr(qpos.contiguous()), nq, _ptr(self.pos), _ptr(self.perm), self.n, self.n_own,
                                 _ptr(self.dense), self.nc_c, _ptr(knn), _ptr(cand), _stream()), "nbk_kd_query")
        return knn


def kth_distance2(comm, q, N, margin):
    """the squared 8th distance of every local row of unit positions q (double, (n, 3)) among the N rows of all ranks;
    and statistics: candidates tested, rows that needed phase 2 and phase-2 queries run, on this rank"""
    P = comm.size
    dev = q.device
    n = int(q.shape[0])
    stats = {'candidates': 0, 'phase2_rows': 0, 'phase2_queries': 0}
    ncell = _ncell(N)
    stats['ncell'] = ncell[0]
    cand = torch.zeros(1, dtype=torch.int64, device=dev)
    if P == 1:
        if n == 0:
            return torch.zeros(0, dtype=torch.float64, device=dev), stats
        with stage("kd_cells"):
            grid = _Grid(q, n, ncell)
        with stage("kd_self"):
            kth = grid.self_kth(cand)
        stats['candidates'] = int(cand.item())
        return kth, stats

    with stage("kd_route"):
        route = _SlabRoute(comm, q, N, margin)
    ntot = int(route.allq.shape[0])
    if ntot >= (1 << 31):
        raise ValueError("KDDensity: %d rows and copies on one rank; at most 2^31 - 1 are supported" % ntot)
    n_own = route.n_own
    grid = None
    kth = torch.zeros(n_own, dtype=torch.float64, device=dev)
    if n_own:
        with stage("kd_cells"):
            grid = _Grid(route.allq, n_own, ncell)
        with stage("kd_self"):
            kth = grid.self_kth(cand)
    del route.allq

    with stage("kd_phase2"):
        own = route.allq_own
        # exact when no row beyond the copies can be nearer: the x-distance to the outer edge of the copies
        if route.full:
            todo = torch.zeros(n_own, dtype=torch.bool, device=dev)
        else:
            x = own[:, 0]
            reach = torch.minimum(x - (route.x0 - route.h), (route.x1 + route.h) - x) - 1e-12
            reach = torch.clamp(reach, min=0.0)
            todo = ~(kth <= reach * reach)
        U = torch.nonzero(todo).reshape(-1)
        nu = int(U.shape[0])
        if int(comm.allreduce(nu)) > 0:
            qU = own.index_select(0, U).contiguous()
            R = torch.sqrt(kth.index_select(0, U))
            rq, send = _route_queries(comm, qU, R)
            Q = torch.cat([qU, rq]) if rq.shape[0] else qU
            K = int(lib().nbk_kd_k())
            if grid is not None:
                knn = grid.query(Q, cand)
            else:
                knn = torch.full((int(Q.shape[0]), K), numpy.inf, dtype=torch.float64, device=dev)
            back = send.back(knn[nu:])
            # the 8th smallest of the owner's list and every returned list
            merged = torch.full((nu, (P + 1) * K), numpy.inf, dtype=torch.float64, device=dev)
            merged[:, :K] = knn[:nu]
            if back.shape[0]:
                cols = (send.dest + 1).reshape(-1, 1) * K + torch.arange(K, device=dev).reshape(1, -1)
                merged[send.src.reshape(-1, 1).expand(-1, K), cols] = back
            kth[U] = torch.sort(merged, dim=1).values[:, K - 1]
            stats['phase2_rows'] = nu
            stats['phase2_queries'] = int(Q.shape[0])
    stats['candidates'] = int(cand.item())
    with stage("kd_back"):
        out = route.back(kth, n)
    return out, stats


class _SlabRoute(object):
    """rows moved to the x slab of the unit box that holds them, plus copies of those within h of a remote slab"""

    def __init__(self, comm, q, N, margin):
        P = comm.size
        dev = q.device
        n = int(q.shape[0])
        pm = ParticleMesh(BoxSize=numpy.ones(3), Nmesh=[P, P, P], dtype='f8', comm=comm)
        self.x0 = pm.x_start / float(P)
        self.x1 = (pm.x_start + pm.x_n) / float(P)
        # owners: the rows listed by the zero-reach routing are remote, all others stay
        self.lay1 = pm._decompose_device(q, 0.0)
        keep = torch.ones(n, dtype=torch.bool, device=dev)
        if self.lay1.ghosts.numel():
            keep[(self.lay1.ghosts & 0xffffffff)] = False
        self.keep = torch.nonzero(keep).reshape(-1)
        recv, _, self.sidx1 = self.lay1.route(q, want_index=True)
        own = torch.cat([q.index_select(0, self.keep), recv]).contiguous()
        self.n_own = int(own.shape[0])
        # copies within h of a remote slab, widened a little so that the rounding of x P can never drop a needed copy;
        # a reach of P + 1 slabs already reaches every slab
        self.h = margin * (1.0 / max(N, 1)) ** (1 / 3.)
        smoothing = min(self.h * P * (1 + 1e-6) + 1e-9, P + 1.0)
        self.full = 2 * self.h + 1.0 / P >= 1.0
        lay2 = pm._decompose_device(own, smoothing)
        cq, _ = lay2.route(own)
        self.allq_own = own
        self.allq = torch.cat([own, cq]).contiguous()

    def back(self, values, n):
        """per-row results of the owned rows to the source's rows"""
        nk = int(self.keep.shape[0])
        o = torch.zeros(n, dtype=values.dtype, device=values.device)
        o[self.keep] = values[:nk]
        self.lay1.gather_back(values[nk:], self.sidx1, o)
        return o


class _QueryRoute(object):
    """phase-2 queries sent to the ranks of `dest` (one row of `src` per entry, grouped by rank)"""

    def __init__(self, comm, src, dest, sendcounts, recvcounts):
        self.comm, self.src, self.dest = comm, src, dest
        self.sendcounts, self.recvcounts = sendcounts, recvcounts

    def back(self, values):
        """per-query results of the received queries (received order) to the sender, in send order"""
        out = torch.empty((int(sum(self.sendcounts)),) + tuple(values.shape[1:]), dtype=values.dtype, device=values.device)
        self.comm.all_to_all_single(out, values.contiguous(), list(self.sendcounts), list(self.recvcounts))
        return out


def _route_queries(comm, qU, R):
    """send every query row to each remote slab within its distance R, widened as the copies are: (the queries received,
    the route back)"""
    P, rank = comm.size, comm.rank
    dev = qU.device
    x = qU[:, 0]
    r = R * (1 + 1e-6) + 1e-9
    src, dest, counts = [], [], []
    for s in range(P):
        if s == rank:
            counts.append(0)
            continue
        a, b = s / float(P), (s + 1) / float(P)
        # periodic distance from x to the slab [a, b)
        g = torch.clamp(torch.maximum(a - x, x - b), min=0.0)
        g = torch.minimum(g, torch.minimum(torch.clamp(torch.maximum(a - (x - 1.0), (x - 1.0) - b), min=0.0),
                                           torch.clamp(torch.maximum(a - (x + 1.0), (x + 1.0) - b), min=0.0)))
        idx = torch.nonzero(g <= r).reshape(-1)
        src.append(idx)
        dest.append(torch.full_like(idx, s))
        counts.append(int(idx.shape[0]))
    src = torch.cat(src) if src else torch.zeros(0, dtype=torch.int64, device=dev)
    dest = torch.cat(dest) if dest else torch.zeros(0, dtype=torch.int64, device=dev)
    recvcounts = comm.alltoall_ints(counts)
    send = qU.index_select(0, src).contiguous()
    recv = torch.empty((int(sum(recvcounts)), 3), dtype=qU.dtype, device=dev)
    comm.all_to_all_single(recv, send, list(recvcounts), list(counts))
    return recv, _QueryRoute(comm, src, dest, counts, recvcounts)
