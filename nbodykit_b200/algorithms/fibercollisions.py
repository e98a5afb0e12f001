"""
Fiber collisions (API of nbodykit/algorithms/fibercollisions.py: FiberCollisions) on one or several GPUs.

Contract (DESIGN.md 4.11).  pos = SkyToUnitSphere(ra, dec) + 1.1; the collision groups are FOF(pos, rad, nmin=1,
absolute=True) in a periodic box of 2.2 (links d^2 <= rad^2 in double).  A group of 2 loses one member, picked without a
distance test; its NeighborID is the other member.  In a group of 3 or more, members collide when
sqrt((dx^2 + dy^2) + dz^2) <= rad in double from the positions cast to float32, and a greedy removes, among the alive
members with the most alive colliders (n_coll) and then the fewest colliders of those colliders (n_other), one pick; the
removed member is collided when its n_coll > 0.  A collided row's NeighborID is the global row of the nearest uncollided
member of its group (the first in member order on a tie).

Every pick comes from a counter-based hash: SplitMix64 of (seed, the group's smallest global row, the removals made in
the group so far) picks the ((h >> 32) k) >> 32-th of the k candidates, members in ascending global row.  The result is
the same for any number of ranks and any split of the rows.

Several GPUs: after FOF, the grouped rows travel to rank label % P, are solved there and their results travel back.
"""
import logging
import math

import numpy
import torch

from .. import CurrentMPIComm
from .._lib import check, lib, stage
from ..pmesh.pm import _ptr, _stream, as_device_tensor
from .fof import FOF, _cells, _sort_rows

_BOX = 2.2
_MASK64 = (1 << 64) - 1


def _mix(z):
    """SplitMix64 finaliser on Python ints (the kernels' fc_mix)"""
    z = (z + 0x9E3779B97F4A7C15) & _MASK64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _MASK64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _MASK64
    return z ^ (z >> 31)


def hash_pick(seed, g, step, k):
    """which of k candidates (in member order) removal `step` of the group whose smallest global row is g removes"""
    h = _mix(_mix(_mix(int(seed)) ^ int(g)) ^ int(step))
    return ((h >> 32) * int(k)) >> 32


def _values(x, name):
    """an ra / dec input (array, Column or tensor) as a one-dimensional NumPy array or tensor"""
    if hasattr(x, "materialize"):
        x = x.materialize()
    if hasattr(x, "compute"):
        x = x.compute()
    if not isinstance(x, torch.Tensor):
        x = numpy.asarray(x)
    if x.ndim != 1:
        raise ValueError("FiberCollisions: %s must be one-dimensional (got shape %s)" % (name, str(tuple(x.shape))))
    return x


def _nonfinite(x):
    if isinstance(x, torch.Tensor):
        return int((~torch.isfinite(x)).sum().item()) if x.is_floating_point() else 0
    return int((~numpy.isfinite(x)).sum()) if x.dtype.kind == 'f' else 0


class FiberCollisions(object):
    """
    Run an angular FOF to find the fiber collision groups of a catalogue, then assign fibers so that as many objects as
    possible receive one (Guo et al. 2012).  Runs on construction.

    - population 1: the largest "clean" sample, in which no two objects collide;
    - population 2: the collided objects.

    Parameters
    ----------
    ra, dec : array_like
        the sky coordinates of the local rows (NumPy arrays, tensors or catalogue columns)
    collision_radius : float, optional
        the angular collision radius in degrees, always (default 62 arcseconds)
    seed : int, optional
        the seed of the fiber choices, in [0, 2^32); None draws one on rank 0 and broadcasts it
    degrees : bool, optional
        whether ``ra`` and ``dec`` are in degrees (else radians)

    Divergences from the reference: every random choice is the hashed pick described in the module documentation, so
    the result does not depend on the number of ranks (the reference draws from NumPy's global generator, group by group
    on each rank); equal-size FOF groups are labelled by their smallest global row; invalid arguments raise
    ``ValueError``.

    Attributes
    ----------
    source : ArrayCatalog
        ``Position`` (the unit-sphere positions + 1.1) with ``BoxSize`` [2.2, 2.2, 2.2]
    labels : ArrayCatalog
        ``Label`` (FOF label, 0 for rows in no group), ``Collided`` (int32 0/1) and ``NeighborID`` (int32 global row of
        the nearest uncollided member of the group, -1 for rows not collided), in the input row order
    attrs : dict
        ``collision_radius``, ``seed`` and ``degrees``
    """
    logger = logging.getLogger('FiberCollisions')

    @CurrentMPIComm.enable
    def __init__(self, ra, dec, collision_radius=62 / 60. / 60., seed=None, degrees=True, comm=None):
        from ..source.catalog.array import ArrayCatalog
        from ..transform import SkyToUnitSphere

        ra_h, dec_h = _values(ra, "ra"), _values(dec, "dec")
        if len(ra_h) != len(dec_h):
            raise ValueError("FiberCollisions: ra and dec have different lengths (%d and %d)" % (len(ra_h), len(dec_h)))
        bad = int(comm.allreduce(_nonfinite(ra_h) + _nonfinite(dec_h)))
        if bad:
            raise ValueError("FiberCollisions: ra and dec must be finite (%d non-finite values)" % bad)
        if not (numpy.isscalar(collision_radius) and numpy.isfinite(float(collision_radius)) and float(collision_radius) > 0):
            raise ValueError("FiberCollisions: collision_radius must be positive and finite (got %r)" % (collision_radius,))
        if seed is not None:
            if isinstance(seed, bool) or not isinstance(seed, (int, numpy.integer)) or not (0 <= int(seed) < (1 << 32)):
                raise ValueError("FiberCollisions: seed must be an integer in [0, 2^32) (got %r)" % (seed,))
        csize = int(comm.allreduce(len(ra_h)))
        if csize >= (1 << 31):
            raise ValueError("FiberCollisions: %d rows in all; NeighborID is int32, so at most 2^31 - 1 are supported" % csize)
        rad = float(numpy.deg2rad(collision_radius))
        try:
            _cells([_BOX] * 3, rad)
        except ValueError:
            raise ValueError("FiberCollisions: a collision radius of %g degrees (%g rad) is below the smallest the FOF cell "
                             "grid supports, about %.3g rad" % (collision_radius, rad, _BOX * math.sqrt(3.0) / (1 << 21)))

        if seed is None:
            if comm.rank == 0:
                seed = numpy.random.randint(0, 4294967295)
            seed = comm.bcast(seed)
        seed = int(seed)

        dev = torch.device("cuda", torch.cuda.current_device())
        pos = SkyToUnitSphere(as_device_tensor(ra_h, device=dev), as_device_tensor(dec_h, device=dev), degrees=degrees) + 1.1
        self.source = ArrayCatalog({'Position': pos.reshape(-1, 3).contiguous()}, comm=comm,
                                   BoxSize=numpy.array([_BOX, _BOX, _BOX]))
        self.comm = comm

        self.attrs = {}
        self.attrs['collision_radius'] = collision_radius
        self.attrs['seed'] = seed
        self.attrs['degrees'] = degrees

        self._collision_radius_rad = rad
        if comm.rank == 0:
            self.logger.info("collision radius in degrees = %.4f" % collision_radius)

        self.run()

    def run(self):
        """find the groups and assign the fibers; sets :attr:`labels`"""
        from ..source.catalog.array import ArrayCatalog
        comm = self.comm
        with stage("fc_fof"):
            fof = FOF(self.source, self._collision_radius_rad, 1, absolute=True)
        label = fof._labels_dev
        pos = self.source['Position'].compute()
        n = int(label.shape[0])
        base = int(fof._offset)
        collided, neighbor, self._stats = assign_fibers(comm, pos, label, base, self._collision_radius_rad,
                                                        self.attrs['seed'])
        self._stats['groups'] = int(fof._nlabels) - 1
        coll = collided.cpu().numpy()
        N_pop2 = int(comm.allreduce(int(coll.sum())))
        N_pop1 = int(self.source.csize) - N_pop2
        f = N_pop2 * 1. / (N_pop1 + N_pop2) if N_pop1 + N_pop2 else 0.0
        if comm.rank == 0:
            self.logger.info("population 1 (clean) size = %d" % N_pop1)
            self.logger.info("population 2 (collided) size = %d" % N_pop2)
            self.logger.info("collision fraction = %.4f" % f)
        data = {'Label': fof.labels, 'Collided': coll, 'NeighborID': neighbor.to(torch.int32).cpu().numpy()}
        assert len(data['Label']) == n
        self.labels = ArrayCatalog(data, comm=comm, **self.source.attrs)


def assign_fibers(comm, pos, label, base, rad, seed):
    """Collided (int32) and NeighborID (int64) of the local rows, from their positions (device, (n, 3)), FOF labels and
    the global row of the first local row; and statistics of this rank's groups"""
    P = comm.size
    dev = label.device
    n = int(label.shape[0])
    with stage("fc_route"):
        rows = torch.nonzero(label > 0).reshape(-1)
        pos4 = pos.index_select(0, rows).to(torch.float32).contiguous()
        lab = label.index_select(0, rows).to(torch.int64)
        grow = rows + base
        if P > 1:
            dest = lab % P
            order = torch.sort(dest, stable=True).indices
            sendcounts = torch.bincount(dest, minlength=P).cpu().tolist()
            recvcounts = comm.alltoall_ints(sendcounts)
            m = int(sum(recvcounts))

            def send(t):
                out = torch.empty((m,) + tuple(t.shape[1:]), dtype=t.dtype, device=dev)
                comm.all_to_all_single(out, t.index_select(0, order).contiguous(), recvcounts, sendcounts)
                return out
            pos4, lab, grow = send(pos4), send(lab), send(grow)
    coll_g, nb_g, stats = _solve(pos4, lab, grow, rad, seed)
    with stage("fc_route"):
        if P > 1:
            def back(t):
                out = torch.empty(len(order), dtype=t.dtype, device=dev)
                comm.all_to_all_single(out, t.contiguous(), sendcounts, recvcounts)
                res = torch.empty_like(out)
                res[order] = out
                return res
            coll_g, nb_g = back(coll_g), back(nb_g)
        collided = torch.zeros(n, dtype=torch.int32, device=dev)
        neighbor = torch.full((n,), -1, dtype=torch.int64, device=dev)
        collided[rows] = coll_g
        neighbor[rows] = nb_g
    return collided, neighbor, stats


def _solve(pos4, lab, grow, rad, seed):
    """the fibers of whole groups: rows in ascending global row (float32 positions, labels > 0, global rows); returns
    (collided, neighbor) in that order and statistics"""
    dev = lab.device
    m = int(lab.shape[0])
    stats = dict(pairs=0, multiplets=0, largest=0, collided=0, steps=0, list_entries=0, candidates=0, rows=m)
    if m == 0:
        return (torch.zeros(0, dtype=torch.int32, device=dev), torch.zeros(0, dtype=torch.int64, device=dev), stats)
    L = lib()
    s = _stream()
    with stage("fc_sort"):
        # a stable sort by label keeps ascending global rows inside every group
        kb = 8 if int(lab.max().item()) >= (1 << 31) else 4
        keys = lab if kb == 8 else lab.to(torch.int32)
        skeys, perm = _sort_rows(keys.clone(), kb, max(1, int(lab.max().item()).bit_length()))
        perm = perm.to(torch.int64)
        pos_s = pos4.index_select(0, perm).contiguous()
        grow_s = grow.index_select(0, perm).contiguous()
        _, size = torch.unique_consecutive(skeys, return_counts=True)
        del skeys
        gstart = torch.zeros(int(size.shape[0]) + 1, dtype=torch.int64, device=dev)
        torch.cumsum(size, 0, out=gstart[1:])
        pairs = torch.nonzero(size == 2).reshape(-1).to(torch.int32)
        W = int(L.nbk_fc_warp_members())
        small = torch.nonzero((size > 2) & (size <= W)).reshape(-1).to(torch.int32)
        large = torch.nonzero(size > W).reshape(-1)
    stats['pairs'] = int(pairs.shape[0])
    stats['multiplets'] = int(small.shape[0]) + int(large.shape[0])
    stats['largest'] = int(size.max().item())
    collided = torch.zeros(m, dtype=torch.int32, device=dev)
    neighbor = torch.full((m,), -1, dtype=torch.int64, device=dev)
    steps = torch.zeros(1, dtype=torch.int64, device=dev)
    seed = int(seed)
    with stage("fc_small"):
        check(L.nbk_fc_pairs(_ptr(gstart), _ptr(pairs), int(pairs.shape[0]), _ptr(grow_s), seed, _ptr(collided), _ptr(neighbor), s),
              "nbk_fc_pairs")
        check(L.nbk_fc_small(_ptr(pos_s), _ptr(gstart), _ptr(small), int(small.shape[0]), _ptr(grow_s), float(rad), seed,
                             _ptr(collided), _ptr(neighbor), _ptr(steps), s), "nbk_fc_small")
    if int(large.shape[0]):
        _solve_large(pos_s, gstart, large, grow_s, rad, seed, collided, neighbor, steps, stats)
    stats['steps'] = int(steps.item())
    stats['collided'] = int(collided.sum().item())
    out_c = torch.empty_like(collided)
    out_n = torch.empty_like(neighbor)
    out_c[perm] = collided
    out_n[perm] = neighbor
    return out_c, out_n, stats


def _solve_large(pos_s, gstart, large, grow_s, rad, seed, collided, neighbor, steps, stats):
    """the groups above one warp: cell-sorted members, CSR collision lists, one block per group, ring-walk neighbours"""
    L = lib()
    s = _stream()
    dev = pos_s.device
    nlg = int(large.shape[0])
    with stage("fc_lists"):
        lseg = gstart.index_select(0, large).contiguous()
        lsize = gstart.index_select(0, large + 1) - lseg
        lbeg = torch.zeros(nlg + 1, dtype=torch.int64, device=dev)
        torch.cumsum(lsize, 0, out=lbeg[1:])
        nl = int(lbeg[-1].item())
        lq64 = torch.repeat_interleave(torch.arange(nlg, dtype=torch.int64, device=dev), lsize)
        lrow = (lseg.index_select(0, lq64) + (torch.arange(nl, dtype=torch.int64, device=dev) - lbeg.index_select(0, lq64))).contiguous()
        lq = lq64.to(torch.int32).contiguous()
        # cells of side >= rad, so that colliding members lie in neighbouring cells
        nc = max(1, int(math.floor(_BOX / (rad * (1 + 1e-6)))))
        cs = _BOX / nc
        keys = torch.empty(nl, dtype=torch.int64, device=dev)
        check(L.nbk_fc_cell_keys(_ptr(pos_s), _ptr(lrow), nl, cs, nc, _ptr(keys), s), "nbk_fc_cell_keys")
        del lrow
        # by cell, then (stably) by group: the members of every group in cell order, at the group's own range
        skeys, p1 = _sort_rows(keys, 8, max(1, (nc * nc * nc - 1).bit_length()))
        p1 = p1.to(torch.int64)
        sq, p2 = _sort_rows(lq.index_select(0, p1).contiguous(), 4, max(1, (nlg - 1).bit_length()))
        del sq
        p2 = p2.to(torch.int64)
        cidx = p1.index_select(0, p2).to(torch.int32).contiguous()
        ckey = skeys.index_select(0, p2).contiguous()
        del skeys, p1, p2
        counts = torch.empty(nl, dtype=torch.int64, device=dev)
        cand = torch.zeros(1, dtype=torch.int64, device=dev)
        check(L.nbk_fc_count(_ptr(pos_s), _ptr(lq), _ptr(lbeg), _ptr(lseg), nl, _ptr(cidx), _ptr(ckey), cs, nc, float(rad),
                             _ptr(counts), _ptr(cand), s), "nbk_fc_count")
        off = torch.zeros(nl + 1, dtype=torch.int64, device=dev)
        torch.cumsum(counts, 0, out=off[1:])
        del counts
        ne = int(off[-1].item())
        nbr = torch.empty(max(ne, 1), dtype=torch.int32, device=dev)
        check(L.nbk_fc_write(_ptr(pos_s), _ptr(lq), _ptr(lbeg), _ptr(lseg), nl, _ptr(cidx), _ptr(ckey), cs, nc, float(rad),
                             _ptr(off), _ptr(nbr), s), "nbk_fc_write")
    stats['list_entries'] = ne
    stats['candidates'] = int(cand.item())
    with stage("fc_greedy"):
        maxn = int(lsize.max().item())
        big = maxn > int(L.nbk_fc_smem_members())
        sc_n = torch.empty(nl if big else 0, dtype=torch.int32, device=dev)
        sc_o = torch.empty(nl if big else 0, dtype=torch.int64, device=dev)
        sc_a = torch.empty(nl if big else 0, dtype=torch.uint8, device=dev)
        nunc = torch.empty(nlg, dtype=torch.int64, device=dev)
        check(L.nbk_fc_greedy(_ptr(lbeg), _ptr(lseg), nlg, maxn, _ptr(off), _ptr(nbr), _ptr(grow_s), seed,
                              _ptr(sc_n) if big else None, _ptr(sc_o) if big else None, _ptr(sc_a) if big else None,
                              _ptr(collided), _ptr(nunc), _ptr(steps), s), "nbk_fc_greedy")
        del sc_n, sc_o, sc_a, nbr, off
    with stage("fc_nearest"):
        check(L.nbk_fc_nearest(_ptr(pos_s), _ptr(lq), _ptr(lbeg), _ptr(lseg), nl, _ptr(cidx), _ptr(ckey), cs, nc,
                               _ptr(collided), _ptr(nunc), _ptr(grow_s), _ptr(neighbor), s), "nbk_fc_nearest")
