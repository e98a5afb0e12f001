"""
Cylindrical groups of centrals and satellites (API of nbodykit/algorithms/cgm.py, Okumura et al. 2017) on one or
several GPUs.

Contract (DESIGN.md 4.9).  The priority of a row is its position 0 .. N-1 in the ascending lexicographic order of the
`rankby` columns, ties by ascending global row index (base/ordering.py); a larger number is a higher priority.  Rows
a != b, a the higher priority, are linked when rsky2 <= rperp^2 and rlos2 <= rpar^2, computed in double from the stored
positions (periodic: wrapped with `pos % L` in their own dtype first): dr = x_a - x_b per axis (periodic: dr > L/2 ->
dr - L, dr <= -L/2 -> dr + L), dr2 = (dx^2 + dy^2) + dz^2, rlos2 = t^2 with t = (dx lx + dy ly) + dz lz for a flat-sky
line of sight l, or with c = (x_a + x_b) / 2, t = (dx cx + dy cy) + dz cz and rlos2 = t^2 / ((cx^2 + cy^2) + cz^2) for
the observer at the origin (no link when that denominator is 0), and rsky2 = |dr2 - rlos2|.  The groups are those of
the greedy of the reference's tests: the highest-priority unassigned row becomes a central, every unassigned row
linked to it its satellite, repeat.

The kernels (csrc/cgm.cu) list each row's higher-priority neighbours on the cell grid of the pair counts, then resolve
the greedy in rounds: a row is a central iff none of its higher-priority neighbours is a central, and a satellite
belongs to the highest-priority central among them.

Several GPUs: x slabs of the box (non-periodic: of the global x range).  Every row moves to the slab that holds it,
copies of the rows within rmax = sqrt(rperp^2 + rpar^2) of a remote slab travel there with their priority, and after
every round the owners' states travel to their copies, until no rank has an undecided row.
"""
import logging
import math
import warnings

import numpy
import torch

from .._lib import check, darr, iarr, lib, stage
from ..base.ordering import check_no_nan, global_rank, key_tensor
from ..pmesh.pm import ParticleMesh, _ptr, _stream
from .fof import _column
from .paircount import _CELLS_PER_SMAX, _Cells

# the per-row states of csrc/cgm.cu (0: undecided)
_CENTRAL, _SATELLITE = 1, 2


class CylindricalGroups(object):
    """
    Compute groups of objects using a cylindrical grouping method: every satellite lies within a cylinder around its
    central.  Runs on construction; the result is :attr:`groups`.

    Parameters
    ----------
    source : CatalogSource
        the input catalogue, with a 'Position' column
    rankby : str, list, ``None``
        the column(s) that rank the objects; objects ranked last (largest values) become centrals first.  ``None``
        ranks by the global row index
    rperp : float
        the radius of the cylinder in the sky plane (perpendicular to the line of sight)
    rpar : float
        half the height of the cylinder along the line of sight
    flat_sky_los : 3-vector, optional
        a fixed unit line-of-sight vector, e.g. [0, 0, 1]; ``None`` takes each pair's own line of sight from the
        observer at the origin
    periodic : bool, optional
        whether to use periodic boundary conditions
    BoxSize : float, 3-vector, optional
        the size of the box; ``source.attrs['BoxSize']`` takes precedence.  Required when ``periodic``

    Divergences from the reference:

    - distances are computed in double from the stored positions; the reference computes them in the positions' own
      dtype, so float32 input can differ at the cylinder's edge;
    - float keys are ordered by value; the reference orders float64 keys by their int64 bit patterns, which reverses
      the order of negative keys;
    - ties of the keys are broken by the global row index; the reference leaves their order to mpsort;
    - periodic positions are wrapped with ``pos % L`` first.

    Memory: per row of a rank, the cell sort of the pair counts, the sorted double positions, 8 bytes of priority, 8 of
    list offsets and 4 bytes per higher-priority neighbour (110 - 150 bytes per row at peak in DESIGN.md 4.9).  On
    several ranks the priority needs (8 K + 8) bytes per row of the whole catalogue for K keys.  At most 2^31 - 1 rows
    per rank, copies included.

    Attributes
    ----------
    groups : ArrayCatalog
        the local rows, in the source's order: ``cgm_type`` ('u4', 0 central, 1 satellite), ``cgm_haloid`` ('i8', for
        a central the number of centrals of higher priority, for a satellite its central's) and ``num_cgm_sats``
        ('i8', a central's number of satellites, 0 for a satellite)
    rounds : int
        the resolution rounds the greedy took
    """
    logger = logging.getLogger('CylindricalGroups')

    def __init__(self, source, rankby, rperp, rpar, flat_sky_los=None, periodic=False, BoxSize=None):
        if 'Position' not in source:
            raise ValueError("the 'Position' column must be defined in the input source")
        if rankby is None:
            rankby = []
        if isinstance(rankby, str):
            rankby = [rankby]
        for col in rankby:
            if col not in source:
                raise ValueError("cannot rank by column '%s'; no such column" % col)

        self.source = source
        self.comm = source.comm
        self.attrs = {}

        self.attrs['BoxSize'] = numpy.empty(3)
        BoxSize = source.attrs.get('BoxSize', BoxSize)
        if periodic and BoxSize is None:
            raise ValueError("please specify a BoxSize if using periodic boundary conditions")
        self.attrs['BoxSize'][:] = BoxSize if BoxSize is not None else numpy.nan

        if flat_sky_los is not None:
            if numpy.isscalar(flat_sky_los) or len(flat_sky_los) != 3:
                raise ValueError("line-of-sight ``flat_sky_los`` should be vector with length 3")
            if not numpy.allclose(numpy.einsum('i,i', flat_sky_los, flat_sky_los), 1.0, rtol=1e-5):
                raise ValueError("line-of-sight ``flat_sky_los`` must be a unit vector")

        for name, v in (('rperp', rperp), ('rpar', rpar)):
            if not (numpy.isscalar(v) and numpy.isfinite(float(v)) and float(v) >= 0):
                raise ValueError("``%s`` must be a non-negative finite number (got %r)" % (name, v))
        if float(rperp) == 0 and float(rpar) == 0:
            raise ValueError("``rperp`` and ``rpar`` cannot both be 0")
        if source.size >= (1 << 31):
            raise ValueError("CylindricalGroups: %d rows on one rank; at most 2^31 - 1 are supported" % source.size)
        if periodic and not numpy.all(numpy.isfinite(self.attrs['BoxSize']) & (self.attrs['BoxSize'] > 0)):
            raise ValueError("the BoxSize of a periodic box must be positive and finite")

        if flat_sky_los is None and periodic:
            warnings.warn(("CylindricalGroups using periodic boundary conditions "
                           "with line-of-sight computed from origin (0,0,0); maybe specify a line-of-sight?"))

        self.attrs['rpar'] = rpar
        self.attrs['rperp'] = rperp
        self.attrs['periodic'] = periodic
        self.attrs['rankby'] = rankby
        self.attrs['flat_sky_los'] = flat_sky_los

        if self.comm.rank == 0:
            self.logger.info("finding groups with rperp=%s and rpar=%s " % (str(rperp), str(rpar)))
        self.run()

    def run(self):
        """compute the groups; sets :attr:`groups` and :attr:`rounds`"""
        from ..source.catalog.array import ArrayCatalog
        comm = self.comm
        P = comm.size
        periodic = bool(self.attrs['periodic'])
        rperp, rpar = float(self.attrs['rperp']), float(self.attrs['rpar'])
        rmax = math.sqrt(rperp * rperp + rpar * rpar)
        los = self.attrs['flat_sky_los']
        los = None if los is None else numpy.asarray(los, dtype='f8').reshape(3)
        box = numpy.asarray(self.attrs['BoxSize'], dtype='f8')

        pos = _column(self.source, 'Position', None)
        if pos.ndim != 2 or pos.shape[1] != 3:
            raise ValueError("CylindricalGroups: Position must have shape (n, 3)")
        dev = pos.device
        n = int(pos.shape[0])
        names = list(self.attrs['rankby'])
        keys = [key_tensor(self.source[k], k) for k in names]
        keys = [k.to(dev) for k in keys]
        for k, name in zip(keys, names):
            if k.shape[0] != n:
                raise ValueError("cannot rank by column '%s': it has %d rows, not %d" % (name, k.shape[0], n))
        check_no_nan(comm, keys, names)
        with stage("cgm_priority"):
            prio = global_rank(comm, keys, n, dev)
            del keys

        with stage("cgm_route"):
            if P > 1:
                route = _SlabRoute(comm, pos, prio, periodic, box, rmax)
                allpos, allprio, n_own = route.allpos, route.allprio, route.n_own
            else:
                route = None
                allpos, allprio, n_own = pos, prio, n
        ntot = int(allpos.shape[0])
        if ntot >= (1 << 31):
            raise ValueError("CylindricalGroups: %d rows and copies on one rank; at most 2^31 - 1 are supported" % ntot)

        types, cen_prio, nsat, stats = _groups(comm, route, allpos, allprio, n_own, periodic, box, los, rperp, rpar)
        self.rounds = stats['rounds']
        self._stats = stats

        with stage("cgm_labels"):
            total = int(comm.allreduce(n)) if P > 1 else n
            flag = torch.zeros(max(total, 1), dtype=torch.uint8, device=dev)
            cen = types == _CENTRAL
            flag[cen_prio[cen]] = 1
            if P > 1:
                comm.allreduce_tensor(flag, "max")
            # haloid of priority p: the centrals above p
            above = flag.flip(0).to(torch.int64).cumsum(0).flip(0) - flag.to(torch.int64)
            haloid = above[cen_prio]
            out_type = (types == _SATELLITE).to(torch.int64)
            out_nsat = torch.where(cen, nsat, torch.zeros_like(nsat))
            if route is not None:
                out_type, haloid, out_nsat = route.back([out_type, haloid, out_nsat], n)
        groups = {'cgm_type': out_type.to(torch.int32).cpu().numpy().astype('u4'),
                  'cgm_haloid': haloid.cpu().numpy().astype('i8'),
                  'num_cgm_sats': out_nsat.cpu().numpy().astype('i8')}
        self.groups = ArrayCatalog(groups, comm=comm, **self.attrs)

        N_cen = int(comm.allreduce(int((groups['cgm_type'] == 0).sum())))
        if comm.rank == 0:
            self.logger.info("found %d CGM centrals total in %d rounds" % (N_cen, self.rounds))


class _SlabRoute(object):
    """rows moved to the x slab that holds them (zero reach), plus copies of those within rmax of a remote slab"""

    def __init__(self, comm, pos, prio, periodic, box, rmax):
        P = comm.size
        dev = pos.device
        n = int(pos.shape[0])
        if periodic:
            rbox = box
            rpos = pos
        else:
            x = pos[:, 0]
            lo = float(x.min().item()) if n else numpy.inf
            hi = float(x.max().item()) if n else -numpy.inf
            lo = min(comm.allgather(lo))
            hi = max(comm.allgather(hi))
            lo = lo if numpy.isfinite(lo) else 0.0
            rbox = numpy.array([hi - lo if hi > lo else 1.0, 1.0, 1.0])
            # slabs of [lo, hi] in double, so that the shift by lo cannot move a row across a slab edge
            rpos = pos.to(torch.float64, copy=True)
            rpos[:, 0] -= lo
        pm = ParticleMesh(BoxSize=rbox, Nmesh=[P, P, P], dtype='f8', comm=comm)
        self.comm = comm
        # owners: the rows listed by the zero-reach routing are remote, all others stay
        self.lay1 = pm._decompose_device(rpos, 0.0)
        keep = torch.ones(n, dtype=torch.bool, device=dev)
        if self.lay1.ghosts.numel():
            keep[(self.lay1.ghosts & 0xffffffff)] = False
        self.keep = torch.nonzero(keep).reshape(-1)
        recv_pos, _, self.sidx1 = self.lay1.route(pos, want_index=True)
        own_pos = torch.cat([pos.index_select(0, self.keep), recv_pos])
        own_prio = torch.cat([prio.index_select(0, self.keep), self.lay1.route_rows(prio, self.sidx1)])
        self.n_own = int(own_pos.shape[0])
        # copies: the owned rows within rmax of a remote slab, widened a little so that the rounding of x P / Lx can
        # never drop a needed copy; a reach of P + 1 slabs already reaches every slab
        if periodic:
            r2 = own_pos
        else:
            r2 = own_pos.to(torch.float64, copy=True)
            r2[:, 0] -= lo
        smoothing = min(rmax * P / float(rbox[0]) * (1 + 1e-6) + 1e-9, P + 1.0)
        self.lay2 = pm._decompose_device(r2, smoothing)
        del r2
        cpos, _, self.sidx2 = self.lay2.route(own_pos, want_index=True)
        cprio = self.lay2.route_rows(own_prio, self.sidx2)
        self.allpos = torch.cat([own_pos, cpos]).contiguous()
        self.allprio = torch.cat([own_prio, cprio]).contiguous()

    def to_copies(self, own_values):
        """per-row values of the owned rows to their copies on the other ranks"""
        return self.lay2.route_rows(own_values, self.sidx2)

    def copies_back(self, copy_values, own):
        """values computed for the copies, added to their owners' `own`"""
        return self.lay2.gather_back(copy_values, self.sidx2, own)

    def back(self, values, n):
        """per-row results of the owned rows to the source's rows"""
        out = []
        nk = int(self.keep.shape[0])
        for v in values:
            o = torch.zeros(n, dtype=v.dtype, device=v.device)
            o[self.keep] = v[:nk]
            self.lay1.gather_back(v[nk:], self.sidx1, o)
            out.append(o)
        return out


def _groups(comm, route, pos, prio, n_own, periodic, box, los, rperp, rpar):
    """the greedy on this rank's owned rows pos[:n_own] (copies after them): per owned row its state, the priority of
    its central, and its satellite count (centrals), in row order; and statistics"""
    dev = pos.device
    n = int(pos.shape[0])
    rmax = math.sqrt(rperp * rperp + rpar * rpar)
    stats = {'rounds': 0, 'candidates': 0, 'neighbours': 0}
    # the cell grid: cells of side >= rmax / 2, as in the pair counts
    with stage("cgm_cells"):
        if n:
            if periodic:
                gbox = box
                origin = numpy.zeros(3)
            else:
                lo = pos.min(0).values.double().cpu().numpy()
                hi = pos.max(0).values.double().cpu().numpy()
                origin = lo
                gbox = numpy.where(hi > lo, hi - lo, 1.0)
            ncell = [int(min(max(1, math.floor(L * _CELLS_PER_SMAX / (rmax * (1 + 1e-4)))), 1 << 20)) for L in gbox]
            # sparse catalogues: wider cells, about 16 rows each at uniform density, so that the CTA of a cell chunk is
            # not mostly idle and the stencil walk visits fewer empty cells
            f = (float(ncell[0]) * ncell[1] * ncell[2] * 16.0 / n) ** (1 / 3.)
            if f > 1:
                ncell = [max(1, int(c / f)) for c in ncell]
            # a row may sit outside its cell by the rounding of its cell index, or by L_f4 - L_f8 when an f4 position
            # wraps to L
            tol = 4e-7 * (numpy.asarray(gbox) + numpy.abs(origin))
            cells = _Cells(pos, torch.zeros(n, dtype=torch.float64, device=dev), periodic, gbox, origin, ncell)
            perm = cells.perm
            perm64 = perm.to(torch.int64)
            sprio = prio.index_select(0, perm64).contiguous()
            first, ckey, nchunks = cells.chunks(int(lib().nbk_cgm_chunk_rows()))
            # sorted position of every row (own rows first) and the owned sorted rows in descending priority
            at = torch.empty(n, dtype=torch.int64, device=dev)
            at[perm64] = torch.arange(n, dtype=torch.int64, device=dev)
            own_sorted = at[:n_own]
            order = own_sorted.index_select(0, torch.argsort(prio[:n_own], descending=True)).to(torch.int32).contiguous()
    state = torch.zeros(max(n, 1), dtype=torch.uint8, device=dev)
    if n:
        geo = (int(periodic), darr(gbox), iarr(ncell), darr(tol), darr(los) if los is not None else None, rperp, rpar)
        with stage("cgm_lists"):
            counts = torch.zeros(n, dtype=torch.int64, device=dev)
            cand = torch.zeros(1, dtype=torch.int64, device=dev)
            check(lib().nbk_cgm_count(_ptr(cells.pos), _ptr(sprio), _ptr(perm), n, n_own, _ptr(first), _ptr(ckey), nchunks,
                                      _ptr(cells.cell_start), _ptr(cells.cell_key), cells.ncells, *geo, _ptr(counts),
                                      _ptr(cand), _stream()), "nbk_cgm_count")
            off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
            torch.cumsum(counts, 0, out=off[1:])
            del counts
            nnb = int(off[-1].item())
            nbr = torch.empty(max(nnb, 1), dtype=torch.int32, device=dev)
            check(lib().nbk_cgm_write(_ptr(cells.pos), _ptr(sprio), _ptr(perm), n, n_own, _ptr(first), _ptr(ckey), nchunks,
                                      _ptr(cells.cell_start), _ptr(cells.cell_key), cells.ncells, *geo, _ptr(off), _ptr(nbr),
                                      _stream()), "nbk_cgm_write")
            stats['candidates'] = int(cand.item())
            stats['neighbours'] = nnb
            del cells, first, ckey
    undecided = torch.zeros(1, dtype=torch.int64, device=dev)
    with stage("cgm_rounds"):
        while True:
            stats['rounds'] += 1
            undecided.zero_()
            if n_own:
                check(lib().nbk_cgm_resolve(_ptr(order), n_own, _ptr(off), _ptr(nbr), _ptr(state), _ptr(undecided), _stream()),
                      "nbk_cgm_resolve")
            if route is None:
                if int(undecided.item()) == 0:
                    break
                continue
            # the owners' states to their copies
            cstate = route.to_copies(state[own_sorted] if n else state[:0])
            if n > n_own:
                state[at[n_own:]] = cstate
            if int(comm.allreduce(int(undecided.item()))) == 0:
                break
    with stage("cgm_assign"):
        cen_prio_s = torch.zeros(max(n, 1), dtype=torch.int64, device=dev)
        nsat_s = torch.zeros(max(n, 1), dtype=torch.int64, device=dev)
        if n_own:
            check(lib().nbk_cgm_assign(_ptr(order), n_own, _ptr(off), _ptr(nbr), _ptr(state), _ptr(sprio), _ptr(cen_prio_s),
                                       _ptr(nsat_s), _stream()), "nbk_cgm_assign")
        if n:
            types = state.index_select(0, own_sorted)
            cen_prio = cen_prio_s.index_select(0, own_sorted)
            nsat = nsat_s.index_select(0, own_sorted)
        else:
            types = state[:0]
            cen_prio = cen_prio_s[:0]
            nsat = nsat_s[:0]
        if route is not None:
            # satellite counts made on copies return to their owners
            ccount = nsat_s.index_select(0, at[n_own:]) if n > n_own else nsat_s[:0]
            route.copies_back(ccount, nsat)
    return types, cen_prio, nsat, stats
