"""
Friends-of-friends halo finder (API of nbodykit/algorithms/fof.py:10-195) on one or several GPUs.

The groups are the connected components of the friend graph: particles i and j are friends when
d^2 = (dx^2 + dy^2) + dz^2 <= b^2, evaluated in double from the positions as stored (periodic: wrapped with `pos % L`
first, per-axis |d| -> min(|d|, L - |d|)).  The local search runs on cells of side <= b / sqrt(3) (csrc/fof.cu): every
pair inside one cell is linked, pairs of cells within reach are merged at their first linked particle pair, and a
lock-free union-find over the cells leaves the smallest global particle id of each group ("minid") at its root.

Several GPUs: x slabs of the box (non-periodic: of the global x range).  Copies of the particles within b of a remote
slab travel there with their global id (the routing of the slab paint), every rank links its own rows plus those
copies, and the `_fof_merge` fixed point of the reference makes the minid of every copy equal.

Labels follow `_assign_labels` (fof.py:197-287): groups with N <= nmin get label 0, the others 1..H by decreasing N.
The one deliberate divergence: the reference orders equal N with NumPy's unstable argsort, which is not reproducible;
here ties are broken by increasing minid, so the same input gives the same labels on any number of GPUs.
"""
import ctypes
import logging
import math

import numpy
import torch

from .._lib import F4, F8, check, darr, iarr, lib, stage
from ..pmesh.pm import ParticleMesh, _ptr, _stream, as_device_tensor

# rows per chunk of the fixed-order segmented reductions of find_features
_CHUNK = 4096
_RED_MIN, _RED_MAX, _RED_SUM = 0, 1, 2


def _code(t):
    return F4 if t.dtype == torch.float32 else F8


def _float_column(col, dev):
    t = as_device_tensor(col, device=dev)
    if t.dtype not in (torch.float32, torch.float64):
        t = t.to(torch.float64)
    return t.contiguous()


def _column(source, name, dev):
    col = source[name]
    if hasattr(col, "materialize"):           # a constant column
        col = col.materialize()
    return _float_column(col.compute() if hasattr(col, "compute") else col, dev)


def _np_mod(x, L):
    """numpy's float `x % L` (fmod, + L where negative) on device tensors"""
    r = torch.fmod(x, L)
    return torch.where(r < 0, r + L, r)


def _cells(extent, b):
    """cells per axis: side extent / n <= b / sqrt(3) with a relative margin, at least one"""
    n = [max(1, int(math.ceil(float(e) * math.sqrt(3.0) * (1.0 + 1e-9) / b))) for e in extent]
    if any(v > (1 << 21) for v in n) or n[0] * n[1] * n[2] >= (1 << 63) - (1 << 53):
        raise ValueError("FOF: %s cells of side b/sqrt(3) do not fit a 63-bit cell key (at most 2^21 per axis); "
                         "the particle extent is too large for this linking length" % str(n))
    return n


def _sort_rows(keys, key_bytes, end_bit):
    """stable radix sort of `keys` (int64 cell keys or int32 labels, all >= 0) carrying the row index along: (sorted keys,
    rows as int32 storage of uint32).  The caller's `keys` buffer is one half of the double buffer; drop it afterwards."""
    n = int(keys.shape[0])
    dev = keys.device
    alt = torch.empty_like(keys)
    rows = torch.empty(n, dtype=torch.int32, device=dev)
    rows_alt = torch.empty_like(rows)
    wb = int(lib().nbk_fof_sort_workspace(n, key_bytes))
    if wb < 0:
        raise ValueError("FOF: cannot sort %d rows" % n)
    work = torch.empty(max(wb, 1), dtype=torch.uint8, device=dev)
    sel = ctypes.c_int(0)
    check(lib().nbk_fof_sort(_ptr(keys), _ptr(alt), _ptr(rows), _ptr(rows_alt), n, key_bytes, int(end_bit), _ptr(work), wb,
                             ctypes.byref(sel), _stream()), "nbk_fof_sort")
    return (alt, rows_alt) if sel.value else (keys, rows)


def _local_fof(pos, gid, gid_base, periodic, box, origin, b, want_minid):
    """union-find over the cells of `pos` (own rows plus received copies).  Returns (row_root: uint32 in int32 storage,
    minid int64 per row or None, cell_min int64, ncells).

    Memory: the sort holds 24 bytes per row (two 8-byte key and two 4-byte row buffers); then sorted keys + rows (12),
    the cell table sized after counting the occupied cells (12 per cell), sorted positions (12 in f4) and the
    union-find (12 per cell): at most ~40 bytes per row when every row has its own cell."""
    dev = pos.device
    n = int(pos.shape[0])
    code = _code(pos)
    if n == 0:
        z = torch.zeros(0, dtype=torch.int64, device=dev)
        return torch.zeros(0, dtype=torch.int32, device=dev), (z.clone() if want_minid else None), z, 0
    ncell = _cells(box, b)
    box_c, org_c, nc_c = darr(box), darr(origin), iarr(ncell)
    with stage("fof_keys"):
        keys = torch.empty(n, dtype=torch.int64, device=dev)
        check(lib().nbk_fof_cell_keys(_ptr(pos), code, n, int(periodic), box_c, org_c, nc_c, float(b), _ptr(keys), _stream()),
              "nbk_fof_cell_keys")
    with stage("fof_sort"):
        end_bit = max(1, (int(ncell[0]) * int(ncell[1]) * int(ncell[2]) - 1).bit_length())
        skeys, perm = _sort_rows(keys, 8, end_bit)
        del keys
    with stage("fof_keys"):
        nw = int(lib().nbk_fof_compact_workspace(n))
        work = torch.empty(nw, dtype=torch.int64, device=dev)
        ncells_d = torch.empty(1, dtype=torch.int64, device=dev)
        check(lib().nbk_fof_compact_count(_ptr(skeys), n, _ptr(work), nw, _ptr(ncells_d), _stream()), "nbk_fof_compact_count")
        ncells = int(ncells_d.item())
        cell_start = torch.empty(ncells + 1, dtype=torch.int32, device=dev)
        cell_key = torch.empty(ncells, dtype=torch.int64, device=dev)
        check(lib().nbk_fof_compact_write(_ptr(skeys), n, _ptr(work), nw, _ptr(cell_start), _ptr(cell_key), _stream()),
              "nbk_fof_compact_write")
        del skeys, work
        spos = torch.empty_like(pos)
        check(lib().nbk_fof_sorted_pos(_ptr(pos), code, n, _ptr(perm), int(periodic), box_c, _ptr(spos), _stream()),
              "nbk_fof_sorted_pos")
    with stage("fof_link"):
        parent = torch.empty(ncells, dtype=torch.int32, device=dev)
        cell_min = torch.empty(ncells, dtype=torch.int64, device=dev)
        check(lib().nbk_fof_link(_ptr(spos), code, _ptr(perm), _ptr(gid), int(gid_base), _ptr(cell_start), _ptr(cell_key), ncells,
                                 int(periodic), box_c, org_c, nc_c, float(b), _ptr(parent), _ptr(cell_min), _stream()),
              "nbk_fof_link")
        del spos, cell_key
    with stage("fof_finalize"):
        row_root = torch.empty(n, dtype=torch.int32, device=dev)
        minid = torch.empty(n, dtype=torch.int64, device=dev) if want_minid else None
        check(lib().nbk_fof_finalize(_ptr(perm), _ptr(cell_start), ncells, _ptr(parent), _ptr(cell_min), _ptr(row_root),
                                     _ptr(minid), _stream()), "nbk_fof_finalize")
    return row_root, minid, cell_min, ncells


class FOF(object):
    """
    A friends-of-friends halo finder that computes the label of each particle, denoting which halo it belongs to
    (Davis et al. 1985).  Runs on construction.

    Parameters
    ----------
    source : CatalogSource
        the source to run the FOF algorithm on; must support 'Position'
    linking_length : float
        the linking length, either in absolute units, or relative to the mean particle separation
    nmin : int
        groups with N <= nmin particles get label 0
    absolute : bool, optional
        If `True`, the linking length is in absolute units, otherwise it is relative to the mean particle separation
    periodic : bool, optional
        link across the faces of ``source.attrs['BoxSize']``
    domain_factor : int, optional
        recorded in :attr:`attrs`; it has no effect, because the decomposition over GPUs is in x slabs

    The cell grid spans the box (periodic) or the bounding box of the particles (non-periodic) with cells of side
    b / sqrt(3), at most 2^21 per axis: a non-periodic catalogue whose extent exceeds ~1.2e6 b on an axis (for instance
    because of one far outlier) raises ValueError.  At most 2^31 - 1 rows per rank.

    Attributes
    ----------
    labels : numpy array ('i4', or 'i8' above 2**31 groups)
        the label of every local row, in the source's row order: 0 for particles in groups of at most `nmin` members,
        else 1..H in order of decreasing group size.  Groups of equal size are ordered by their smallest global
        particle id (the reference leaves that order to an unstable sort).
    max_label : list
        ``comm.allgather(labels.max())``
    """
    logger = logging.getLogger('FOF')

    def __init__(self, source, linking_length, nmin, absolute=False, periodic=True, domain_factor=1):
        self.comm = source.comm
        self._source = source

        if 'Position' not in source:
            raise ValueError("cannot compute FOF without 'Position' column")

        self.attrs = {}
        self.attrs['linking_length'] = linking_length
        self.attrs['nmin'] = nmin
        self.attrs['absolute'] = absolute
        self.attrs['periodic'] = periodic
        self.attrs['domain_factor'] = domain_factor

        if periodic and 'BoxSize' not in source.attrs:
            raise ValueError("Periodic FOF requires BoxSize in .attrs['BoxSize']")

        if not absolute:
            if 'Nmesh' in source.attrs:
                ndim = len(numpy.atleast_1d(source.attrs['Nmesh']))
            else:
                ndim = source['Position'].shape[1]
            mean_separation = pow(numpy.prod(source.attrs['BoxSize']) / source.csize, 1.0 / ndim)
            linking_length *= mean_separation
        self._linking_length = float(linking_length)
        if not (self._linking_length > 0 and numpy.isfinite(self._linking_length)):
            raise ValueError("FOF: the linking length must be positive and finite (got %r)" % self._linking_length)

        self.run()

    # ------------------------------------------------------------------------------------------------------------------
    def _box(self):
        return numpy.ones(3) * numpy.asarray(self._source.attrs['BoxSize'], dtype='f8')

    def run(self):
        """find the groups; sets :attr:`labels` and :attr:`max_label`"""
        comm = self.comm
        P, rank = comm.size, comm.rank
        periodic = bool(self.attrs['periodic'])
        b = self._linking_length
        pos = _column(self._source, 'Position', None)
        if pos.ndim != 2 or pos.shape[1] != 3:
            raise ValueError("FOF: Position must have shape (n, 3)")
        dev = pos.device
        n = int(pos.shape[0])
        if n >= (1 << 31):
            raise ValueError("FOF: %d rows on one rank; at most 2^31 - 1 are supported" % n)
        sizes = comm.allgather(n)
        base = int(sum(sizes[:rank]))
        self._offset = base

        if periodic:
            box = self._box()
            origin = numpy.zeros(3)
        else:
            lo = pos.min(0).values.double().cpu().numpy() if n else numpy.full(3, numpy.inf)
            hi = pos.max(0).values.double().cpu().numpy() if n else numpy.full(3, -numpy.inf)
            lo = numpy.min(comm.allgather(lo), axis=0)
            hi = numpy.max(comm.allgather(hi), axis=0)
            origin = numpy.where(numpy.isfinite(lo), lo, 0.0)
            box = numpy.where(hi > lo, hi - lo, 1.0)

        layout = sidx = None
        with stage("fof_route"):
            if P > 1:
                layout, sidx, rpos, rgid = self._route(pos, periodic, box, origin, base, b)
                allpos = torch.cat([pos, rpos]) if rpos.numel() else pos
                gid = torch.cat([torch.arange(base, base + n, dtype=torch.int64, device=dev), rgid])
            else:
                allpos, gid = pos, None

        row_root, minid, cell_min, ncells = _local_fof(allpos, gid, base, periodic, box, origin, b, P > 1)
        del allpos

        root_min = cell_min
        if P > 1:
            with stage("fof_merge"):
                root_min, self.merge_rounds = self._merge(layout, sidx, n, row_root, minid, ncells)
        else:
            self.merge_rounds = 0

        with stage("fof_labels"):
            self._labels_dev, self._nlabels = self._assign_labels(row_root[:n], root_min, ncells, n, sizes)
        self.labels = self._labels_dev.cpu().numpy()
        self.max_label = comm.allgather(self.labels.max() if self.labels.size else self.labels.dtype.type(0))

    def _route(self, pos, periodic, box, origin, base, b):
        """copies of the rows within b of a remote x slab, with their global ids"""
        comm = self.comm
        P = comm.size
        if periodic:
            rpos_src = pos
            rbox = box
        else:
            rpos_src = pos.clone()
            rpos_src[:, 0] -= origin[0]
            rbox = numpy.array([box[0], 1.0, 1.0])
        pm = ParticleMesh(BoxSize=rbox, Nmesh=[P, P, P], dtype='f8', comm=comm)
        # the reach in slab units, widened a little so that rounding of x * P / Lx can never drop a needed copy
        smoothing = b * P / float(rbox[0]) * (1 + 1e-6) + 1e-9
        if smoothing >= 64:
            raise ValueError("FOF: the linking length spans more than 64 slab widths")
        layout = pm._decompose_device(rpos_src, smoothing)
        del rpos_src
        rpos, _, sidx = layout.route(pos, want_index=True)
        rgid = layout.route_rows(torch.arange(base, base + int(pos.shape[0]), dtype=torch.int64, device=pos.device), sidx)
        return layout, sidx, rpos, rgid

    def _merge(self, layout, sidx, n, row_root, minid, ncells):
        """`_fof_merge` (fof.py:311-337): the owner takes the minimum over its copies, the copies take the owner's value,
        every rank lowers each local component to its smallest value, until no rank changes a row"""
        comm = self.comm
        dev = minid.device
        root_min = torch.empty(max(ncells, 1), dtype=torch.int64, device=dev)
        changed = torch.zeros(1, dtype=torch.int64, device=dev)
        rounds = 0
        while True:
            rounds += 1
            own = minid[:n].clone()
            layout.gather_back_min(minid[n:], sidx, own)
            new = torch.cat([own, layout.route_rows(own, sidx)])
            changed.zero_()
            check(lib().nbk_fof_lower(_ptr(row_root), int(minid.shape[0]), _ptr(new), ncells, _ptr(root_min), _ptr(minid),
                                      _ptr(changed), _stream()), "nbk_fof_lower")
            if int(comm.allreduce(int(changed.item()))) == 0:
                break
        if ncells == 0:
            root_min = root_min[:0]
        return root_min, rounds

    def _assign_labels(self, own_root, root_min, ncells, n, sizes):
        """labels 0 (N <= nmin) and 1..H by (-N, minid), per local row"""
        comm = self.comm
        P = comm.size
        dev = own_root.device
        counts = torch.zeros(max(ncells, 1), dtype=torch.int64, device=dev)
        check(lib().nbk_fof_root_counts(_ptr(own_root), n, _ptr(counts), _stream()), "nbk_fof_root_counts")
        if P == 1:
            # one rank holds whole groups: only those above nmin enter the table (most groups are single particles)
            roots = torch.nonzero(counts[:ncells] > int(self.attrs['nmin'])).reshape(-1)
        else:
            roots = torch.nonzero(counts[:ncells]).reshape(-1)
        gmin, gcnt = root_min[roots], counts[roots]
        del counts, roots
        if P > 1:
            # local components that merged elsewhere share a minid: combine, then send each group to the rank owning its id
            gmin, inv = torch.unique(gmin, return_inverse=True)
            gcnt = torch.zeros(gmin.shape[0], dtype=torch.int64, device=dev).index_add_(0, inv, gcnt)
            bounds = torch.tensor(numpy.cumsum(sizes)[:-1], dtype=torch.int64, device=dev)
            owner = torch.bucketize(gmin, bounds, right=True)
            sendcounts = torch.bincount(owner, minlength=P).cpu().tolist()
            recvcounts = comm.alltoall_ints(sendcounts)
            # gmin is sorted, so the owners are already grouped in rank order
            rmin = torch.empty(sum(recvcounts), dtype=torch.int64, device=dev)
            rcnt = torch.empty_like(rmin)
            comm.all_to_all_single(rmin, gmin, recvcounts, sendcounts)
            comm.all_to_all_single(rcnt, gcnt, recvcounts, sendcounts)
            gmin, inv = torch.unique(rmin, return_inverse=True)
            gcnt = torch.zeros(gmin.shape[0], dtype=torch.int64, device=dev).index_add_(0, inv, rcnt)
        big = gcnt > int(self.attrs['nmin'])
        bmin, bcnt = gmin[big].cpu().numpy(), gcnt[big].cpu().numpy()
        if P > 1:
            parts = comm.allgather((bmin, bcnt))
            bmin = numpy.concatenate([p[0] for p in parts])
            bcnt = numpy.concatenate([p[1] for p in parts])
        order = numpy.lexsort((bmin, -bcnt))            # decreasing N, then increasing minid
        bmin, bcnt = bmin[order], bcnt[order]
        self._group_sizes = bcnt
        H = len(bmin)
        # label of every local root: position in the (minid-sorted) table of the big groups + 1, else 0
        by_id = numpy.argsort(bmin)
        ids = torch.as_tensor(bmin[by_id], dtype=torch.int64, device=dev)
        lab = torch.as_tensor(by_id + 1, dtype=torch.int64, device=dev)
        cell_label = torch.zeros(max(ncells, 1), dtype=torch.int64, device=dev)
        if H and ncells:
            # in slices: the lookup temporaries stay small next to the per-cell arrays
            step = 1 << 26
            for a in range(0, ncells, step):
                rm = root_min[a:a + step]
                j = torch.searchsorted(ids, rm).clamp_(max=H - 1)
                cell_label[a:a + step] = torch.where(ids[j] == rm, lab[j], torch.zeros_like(rm))
        ldt = torch.int64 if H + 1 > 2 ** 31 else torch.int32
        labels = torch.empty(n, dtype=ldt, device=dev)
        check(lib().nbk_fof_label_rows(_ptr(own_root), n, _ptr(cell_label), _ptr(labels), 8 if ldt == torch.int64 else 4,
                                       _stream()), "nbk_fof_label_rows")
        return labels, H + 1

    # ------------------------------------------------------------------------------------------------------------------
    def find_features(self, peakcolumn=None):
        """
        Based on the particle labels, identify the groups, and return the center-of-mass ``CMPosition``, ``CMVelocity``,
        and ``Length`` of each feature (``InitialPosition`` too when the source has it).  If a ``peakcolumn`` is given,
        ``PeakPosition`` and ``PeakVelocity`` are the center of mass of the particles of each group at the maximum of
        that column.  Row 0 collects the particles of label 0 and has ``Length`` 0; its ``PeakPosition`` /
        ``PeakVelocity`` are taken over the label-0 particles at their maximum (the reference pools every non-peak
        particle of every group into row 0 instead).  Rows 1..H follow the reference's formulas.

        The rows are split over the ranks as ScatterArray splits them (rank r gets n // P + (r < n % P) rows).  The
        sums are taken in double in a fixed order, so a run is reproducible bit for bit.  On P > 1 each rank sums its
        own rows and the sums are allreduced (as the reference does): the catalogue equals the single-rank one to the
        float32 rounding of its columns, not bit for bit, while ``Length`` and the labels are identical.

        Returns
        -------
        :class:`~nbodykit_b200.source.catalog.array.ArrayCatalog`
        """
        from ..source.catalog.array import ArrayCatalog
        source = self._source
        for col in ['Position', 'Velocity']:
            if col not in source:
                raise ValueError("the column '%s' is missing from parent source; cannot compute halos" % col)
        if peakcolumn is not None and peakcolumn not in source:
            raise ValueError("the peak column '%s' is missing from parent source" % peakcolumn)
        with stage("fof_features"):
            data = self._features(peakcolumn)
        attrs = source.attrs.copy()
        attrs.update(self.attrs)
        return ArrayCatalog(data, comm=self.comm, **attrs)

    def _features(self, peakcolumn):
        comm = self.comm
        P, rank = comm.size, comm.rank
        periodic = bool(self.attrs['periodic'])
        source = self._source
        labels = self._labels_dev
        dev = labels.device
        n = int(labels.shape[0])
        H1 = int(self._nlabels)
        box = self._box() if periodic else numpy.ones(3)
        box_c = darr(box)
        Lt = torch.as_tensor(box, dtype=torch.float64, device=dev)

        # rows ordered by label (stable radix sort: row order within a label) and fixed chunks of every label's segment
        kb = 8 if labels.dtype == torch.int64 else 4
        srt, order = _sort_rows(labels.clone(), kb, max(1, (H1 - 1).bit_length()))
        seg = torch.searchsorted(srt, torch.arange(H1 + 1, dtype=labels.dtype, device=dev)).to(torch.int64)
        del srt
        nch = (seg[1:] - seg[:-1] + (_CHUNK - 1)) // _CHUNK
        label_chunk = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), torch.cumsum(nch, 0)])
        nchunks = int(label_chunk[-1].item())
        chunk_label = torch.repeat_interleave(torch.arange(H1, dtype=torch.int64, device=dev), nch)
        chunk_first = seg[chunk_label] + (torch.arange(nchunks, dtype=torch.int64, device=dev) - label_chunk[chunk_label]) * _CHUNK
        chunk_first = torch.cat([chunk_first, torch.full((1,), n, dtype=torch.int64, device=dev)])
        partial = torch.empty((max(nchunks, 1), 4), dtype=torch.float64, device=dev)

        def reduce(op, col, ref=None, mask=None, thresh=None, wrap=False, allop="sum"):
            out = torch.empty((H1, 4), dtype=torch.float64, device=dev)
            check(lib().nbk_fof_segment_reduce(op, _ptr(col), _code(col), _ptr(mask), _code(mask) if mask is not None else F8,
                                               _ptr(thresh), _ptr(ref), int(wrap), box_c, _ptr(order), _ptr(chunk_first),
                                               _ptr(chunk_label), nchunks, _ptr(label_chunk), H1, _ptr(partial), _ptr(out),
                                               _stream()), "nbk_fof_segment_reduce")
            if P > 1:
                if allop == "sum":
                    comm.allreduce_tensor(out, "sum")
                else:
                    vals = out[:, :3].contiguous()
                    comm.allreduce_tensor(vals, allop)
                    cnt = out[:, 3].contiguous()
                    comm.allreduce_tensor(cnt, "sum")
                    out = torch.cat([vals, cnt[:, None]], 1)
            return out

        def centre(col, mask=None, thresh=None, is_pos=True):
            """centerofmass (fof.py:647-700): posmin + mean of the wrapped offsets, % L when periodic"""
            if is_pos:
                pmin = reduce(_RED_MIN, col, mask=mask, thresh=thresh, allop="min")[:, :3].contiguous()
                s = reduce(_RED_SUM, col, ref=pmin, mask=mask, thresh=thresh, wrap=periodic)
                c = pmin + s[:, :3] / s[:, 3:4]
                if periodic:
                    c = _np_mod(c, Lt)
            else:
                s = reduce(_RED_SUM, col, mask=mask, thresh=thresh)
                c = s[:, :3] / s[:, 3:4]
            return c, s[:, 3]

        pos = _column(source, 'Position', dev)
        vel = _column(source, 'Velocity', dev)
        hpos, N = centre(pos)
        hvel, _ = centre(vel, is_pos=False)
        cols = {'CMPosition': hpos, 'CMVelocity': hvel}
        if 'InitialPosition' in source:
            cols['InitialPosition'], _ = centre(_column(source, 'InitialPosition', dev))
        if peakcolumn is not None:
            peak = _column(source, peakcolumn, dev).reshape(-1)
            dmax = reduce(_RED_MAX, peak, allop="max")[:, 0].contiguous()
            cols['PeakPosition'], _ = centre(pos, mask=peak, thresh=dmax)
            cols['PeakVelocity'], _ = centre(vel, mask=peak, thresh=dmax, is_pos=False)

        length = N.round().to(torch.int64)
        length[0] = 0
        # ScatterArray's split of the H+1 rows
        lo = rank * (H1 // P) + min(rank, H1 % P)
        hi = lo + H1 // P + (1 if rank < H1 % P else 0)
        out = {}
        for name in ('CMPosition', 'CMVelocity', 'InitialPosition', 'PeakPosition', 'PeakVelocity'):
            if name in cols:
                out[name] = cols[name][lo:hi].to(torch.float32).cpu().numpy()
        out['Length'] = length[lo:hi].to(torch.int32).cpu().numpy()
        return out

    def to_halos(self, particle_mass, cosmo, redshift, mdef='vir', posdef='cm', peakcolumn='Density'):
        """
        A :class:`~nbodykit_b200.source.catalog.halos.HaloCatalog` of the groups (fof.py:130-195): the centre-of-mass
        (``posdef='cm'``) or peak (``posdef='peak'``, the rows at the maximum of ``peakcolumn``) position and velocity of
        every group with members, and ``Mass = particle_mass * Length``, with the analytic default radius and
        concentration at ``cosmo`` and ``redshift`` for the mass definition ``mdef``.

        ``cosmo`` must be this package's :class:`~nbodykit_b200.cosmology.Cosmology`: the reference hands other
        cosmologies (astropy's) to halotools, which is not a dependency.
        """
        from ..cosmology import Cosmology
        from ..source.catalog.array import ArrayCatalog
        from ..source.catalog.halos import HaloCatalog
        if not isinstance(cosmo, Cosmology):
            raise NotImplementedError("FOF.to_halos: a cosmology other than nbodykit_b200's Cosmology (got %r) is handed "
                                      "to halotools by the reference; halotools is not a dependency of nbodykit_b200"
                                      % (cosmo,))
        if posdef not in ('cm', 'peak'):
            raise ValueError("``posdef`` should be 'cm' or 'peak' (got %r)" % (posdef,))
        features = self.find_features(peakcolumn=peakcolumn if posdef == 'peak' else None)
        keep = numpy.asarray(features['Length'].compute()) > 0
        prefix = 'CM' if posdef == 'cm' else 'Peak'
        data = {k: numpy.asarray(features[k].compute())[keep] for k in features.columns
                if k in ('CMPosition', 'CMVelocity', 'InitialPosition', 'PeakPosition', 'PeakVelocity', 'Length')}
        data['Position'] = data[prefix + 'Position']
        data['Velocity'] = data[prefix + 'Velocity']
        data['Mass'] = particle_mass * data['Length']
        attrs = dict(features.attrs)
        attrs['particle_mass'] = particle_mass
        halos = ArrayCatalog(data, comm=self.comm, **attrs)
        return HaloCatalog(halos, cosmo, redshift, mdef=mdef, mass='Mass', position='Position', velocity='Velocity')
