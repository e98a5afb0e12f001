"""
The global order of a catalogue's rows by one or several key columns, shared by `CatalogSource.sort` and
`CylindricalGroups`.

Rows are ordered lexicographically by the keys, the first key primary, each ascending (descending with `reverse`).
Values compare numerically, so -0.0 == 0.0; ties are broken by ascending global row index (local index plus the sizes
of the lower ranks).  A key column must be 1-D and integer or floating point, without NaN.

One rank: stable `torch.sort` passes from the last key to the first.  Several ranks: every rank all-gathers the key
columns (one sum all-reduce of each zero-padded column) and sorts the same table, then keeps the positions of its own
rows.  That holds (8 K + 8) N_total bytes per GPU for K keys and N_total rows in all, plus the sort's scratch.
"""
import numpy
import torch

_INT_DTYPES = (torch.int8, torch.uint8, torch.int16, torch.uint16, torch.int32, torch.uint32, torch.int64, torch.uint64)


def key_tensor(col, name, device=None):
    """a key column as a 1-D int64 or float64 tensor on `device` (None: where it is; host for NumPy columns), with -0.0
    turned into 0.0; raises ValueError for a column that is not 1-D integer or floating point"""
    if hasattr(col, 'materialize'):
        col = col.materialize()
    col = col.compute() if hasattr(col, 'compute') else col
    if isinstance(col, torch.Tensor):
        t = col
        if not (t.is_floating_point() or t.dtype in _INT_DTYPES):
            raise ValueError("cannot sort by column '%s' with dtype '%s'; must be integer or floating type" % (name, t.dtype))
        if t.dtype == torch.uint64:
            t = t.view(torch.int64) ^ torch.tensor(-2 ** 63, dtype=torch.int64, device=t.device)
    else:
        a = numpy.asarray(col)
        if not (numpy.issubdtype(a.dtype, numpy.integer) or numpy.issubdtype(a.dtype, numpy.floating)):
            raise ValueError("cannot sort by column '%s' with dtype '%s'; must be integer or floating type" % (name, a.dtype))
        if a.dtype == numpy.uint64:
            # order-preserving map onto int64
            a = a.view('i8') ^ numpy.int64(-2 ** 63)
        t = torch.from_numpy(numpy.ascontiguousarray(a))
    if t.ndim != 1:
        raise ValueError("cannot sort by column '%s': a key column must be one-dimensional, not of shape %s"
                         % (name, tuple(t.shape)))
    if device is not None:
        t = t.to(device)
    if t.is_floating_point():
        t = t.to(torch.float64)
        t = torch.where(t == 0, torch.zeros_like(t), t)
    else:
        t = t.to(torch.int64)
    return t.contiguous()


def check_no_nan(comm, keys, names):
    """raise ValueError on every rank when any rank holds a NaN key"""
    bad = [int(bool(torch.isnan(k).any().item())) if k.is_floating_point() else 0 for k in keys]
    if comm.size > 1:
        bad = [int(v) for v in numpy.atleast_1d(comm.allreduce(numpy.asarray(bad, dtype='i8')))] if bad else bad
    for v, name in zip(bad, names):
        if v:
            raise ValueError("cannot sort by column '%s': it holds NaN" % name)


def _order_table(keys, n, reverse):
    """rows of the table in key order, ties by ascending row: stable sorts from the last key to the first"""
    dev = keys[0].device if keys else None
    idx = torch.arange(n, dtype=torch.int64, device=dev)
    for k in reversed(keys):
        o = torch.sort(k.index_select(0, idx), stable=True, descending=bool(reverse)).indices
        idx = idx.index_select(0, o)
    return idx


def global_rank(comm, keys, n, device, reverse=False):
    """the position (int64, 0 .. N_total - 1) of each of this rank's `n` rows in the global order of `keys` (tensors
    from `key_tensor`); no keys: the global row index"""
    sizes = comm.allgather(int(n)) if comm.size > 1 else [int(n)]
    base = int(sum(sizes[:comm.rank]))
    total = int(sum(sizes))
    if not keys:
        return torch.arange(base, base + n, dtype=torch.int64, device=device)
    if comm.size > 1:
        table = []
        for k in keys:
            g = torch.zeros(total, dtype=k.dtype, device=k.device)
            g[base:base + n] = k
            comm.allreduce_tensor(g, "sum")
            table.append(g)
    else:
        table = keys
    order = _order_table(table, total, reverse)
    del table
    rank = torch.empty(total, dtype=torch.int64, device=order.device)
    rank[order] = torch.arange(total, dtype=torch.int64, device=order.device)
    return rank[base:base + n].contiguous()
