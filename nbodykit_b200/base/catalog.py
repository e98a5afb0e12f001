"""
CatalogSource -- a table of per-particle columns (API of nbodykit/base/catalog.py on the FFTPower
path: column protocol :269-273,327-404, `compute` :530-560, `to_mesh` :787-873, default columns
`Selection/Weight/Value` :1166-1216, `size/csize` :974-1011).

GPU-first differences from the reference:
  * no dask: a column is a NumPy array (host) or a torch tensor (host or HBM); a catalogue whose
    columns already live on the GPU is painted without any host round trip;
  * the default `Weight`, `Value`, `Selection` columns are `ConstantColumn`s that are never
    materialised -- the scatter kernel is simply launched without a mass pointer.
"""
import logging
import numbers

import numpy
import torch

from .. import CurrentMPIComm


def _is_torch(a):
    return isinstance(a, torch.Tensor)


class Column(object):
    """a per-particle array-like with `.compute()` (the dask-array role in the reference)"""

    def __init__(self, data):
        if isinstance(data, Column):
            data = data.data
        if not _is_torch(data):
            data = numpy.asarray(data)
        self.data = data

    # -- array protocol
    def compute(self):
        return self.data

    @property
    def shape(self):
        return tuple(self.data.shape)

    @property
    def dtype(self):
        if _is_torch(self.data):
            return numpy.dtype(str(self.data.dtype).replace("torch.", ""))
        return self.data.dtype

    @property
    def ndim(self):
        return len(self.shape)

    def __len__(self):
        return self.shape[0]

    def __array__(self, dtype=None, copy=None):
        a = self.data.detach().cpu().numpy() if _is_torch(self.data) else self.data
        return a.astype(dtype) if dtype is not None else a

    def __getitem__(self, idx):
        if isinstance(idx, Column):
            idx = idx.data
        if _is_torch(self.data) and isinstance(idx, numpy.ndarray):
            idx = torch.from_numpy(idx).to(self.data.device)
        return Column(self.data[idx])

    def astype(self, dtype):
        if _is_torch(self.data):
            return Column(self.data.to(getattr(torch, numpy.dtype(dtype).name)))
        return Column(self.data.astype(dtype))

    def sum(self, axis=None):
        """sum of the column (a Python float / array for axis != None); device columns reduce on the device"""
        if _is_torch(self.data):
            r = self.data.double().sum() if axis is None else self.data.double().sum(dim=axis)
            return float(r.item()) if axis is None else r.cpu().numpy()
        return self.data.sum(axis=axis, dtype='f8' if self.data.dtype.kind == 'f' else None)

    def __repr__(self):
        where = ("torch:%s" % self.data.device) if _is_torch(self.data) else "numpy"
        return "Column(shape=%s, dtype=%s, %s)" % (self.shape, self.dtype, where)

    # -- arithmetic (so that e.g. cat['Position'] + cat['Velocity'] * los keeps working)
    def _binary(self, other, op, reverse=False):
        o = other.materialize(len(self), like=self.data) if isinstance(other, ConstantColumn) else \
            (other.data if isinstance(other, Column) else other)
        a = self.data
        if _is_torch(a) and isinstance(o, (numpy.ndarray, list, tuple)):
            o = torch.as_tensor(numpy.asarray(o)).to(a.device)
        elif not _is_torch(a) and _is_torch(o):
            a = torch.from_numpy(numpy.ascontiguousarray(a)).to(o.device)
        return Column(op(o, a) if reverse else op(a, o))

    def __add__(self, o): return self._binary(o, lambda a, b: a + b)
    def __radd__(self, o): return self._binary(o, lambda a, b: a + b, True)
    def __sub__(self, o): return self._binary(o, lambda a, b: a - b)
    def __rsub__(self, o): return self._binary(o, lambda a, b: a - b, True)
    def __mul__(self, o): return self._binary(o, lambda a, b: a * b)
    def __rmul__(self, o): return self._binary(o, lambda a, b: a * b, True)
    def __truediv__(self, o): return self._binary(o, lambda a, b: a / b)
    def __rtruediv__(self, o): return self._binary(o, lambda a, b: a / b, True)
    def __pow__(self, o): return self._binary(o, lambda a, b: a ** b)
    def __mod__(self, o): return self._binary(o, lambda a, b: a % b)
    def __neg__(self): return Column(-self.data)
    def __lt__(self, o): return self._binary(o, lambda a, b: a < b)
    def __le__(self, o): return self._binary(o, lambda a, b: a <= b)
    def __gt__(self, o): return self._binary(o, lambda a, b: a > b)
    def __ge__(self, o): return self._binary(o, lambda a, b: a >= b)
    def __and__(self, o): return self._binary(o, lambda a, b: a & b)
    def __or__(self, o): return self._binary(o, lambda a, b: a | b)
    def __invert__(self): return Column(~self.data)


class ConstantColumn(Column):
    """a column holding one value for every particle without storing it (transform.ConstantArray role,
    nbodykit/transform.py:89-106)"""

    def __init__(self, value, size):
        self.value = value
        self.size = int(size)
        self.data = None

    @property
    def shape(self):
        return (self.size,) + tuple(numpy.shape(self.value))

    @property
    def dtype(self):
        return numpy.asarray(self.value).dtype

    def materialize(self, n=None, like=None):
        n = self.size if n is None else n
        if _is_torch(like):
            v = torch.as_tensor(numpy.asarray(self.value))
            return v.to(like.device).expand((n,) + tuple(v.shape)).clone()
        return numpy.broadcast_to(numpy.asarray(self.value), (n,) + tuple(numpy.shape(self.value))).copy()

    def compute(self):
        return self.materialize()

    def sum(self, axis=None):
        return self.value * self.size

    def __array__(self, dtype=None, copy=None):
        a = self.materialize()
        return a.astype(dtype) if dtype is not None else a

    def __getitem__(self, idx):
        if isinstance(idx, slice):
            return ConstantColumn(self.value, len(range(*idx.indices(self.size))))
        i = idx.data if isinstance(idx, Column) else idx
        if _is_torch(i):
            n = int(i.sum().item()) if i.dtype == torch.bool else int(i.numel())
        else:
            i = numpy.asarray(i)
            n = int(i.sum()) if i.dtype == bool else int(i.size)
        return ConstantColumn(self.value, n)

    def _binary(self, other, op, reverse=False):
        if isinstance(other, ConstantColumn):
            v = op(other.value, self.value) if reverse else op(self.value, other.value)
            return ConstantColumn(v, self.size)
        if isinstance(other, Column):
            return other._binary(self, op, not reverse)
        if numpy.isscalar(other):
            v = op(other, self.value) if reverse else op(self.value, other)
            return ConstantColumn(v, self.size)
        return Column(self.materialize())._binary(other, op, reverse)

    def __neg__(self): return ConstantColumn(-self.value, self.size)
    def __invert__(self): return ConstantColumn(not self.value, self.size)

    def __repr__(self):
        return "ConstantColumn(%r, size=%d)" % (self.value, self.size)


def column(name=None, is_default=False):
    """decorator marking a method as a hard-coded column (base/catalog.py:97-125)"""
    def decorator(getter):
        getter.column_name = name if isinstance(name, str) else getter.__name__
        getter.is_default = is_default
        return getter
    if hasattr(name, '__call__'):
        getter, name = name, None
        return decorator(getter)
    return decorator


def find_column(cls, name):
    """the hard-coded column `name` of a class, searching the MRO"""
    for k in cls.__mro__:
        f = k.__dict__.get(name, None)
        if f is not None and hasattr(f, 'column_name'):
            return f
    return None


def find_columns(cls):
    out = []
    for k in cls.__mro__:
        for key, val in k.__dict__.items():
            if hasattr(val, 'column_name') and val.column_name not in out:
                out.append(val.column_name)
    return sorted(out)


class CatalogSourceBase(object):
    """the column container (base/catalog.py:167-560)"""
    logger = logging.getLogger('CatalogSourceBase')

    def __new__(cls, *args, **kwargs):
        obj = object.__new__(cls)
        obj._overrides = {}
        obj._attrs = {}
        obj.base = None
        return obj

    def __init__(self, comm):
        self.comm = comm
        self.base = None
        if not hasattr(self, '_overrides'):
            self._overrides = {}

    # ---- metadata
    @property
    def attrs(self):
        try:
            return self._attrs
        except AttributeError:
            self._attrs = {}
            return self._attrs

    @property
    def hardcolumns(self):
        return find_columns(self.__class__)

    @property
    def columns(self):
        return sorted(set(self.hardcolumns) | set(self._overrides))

    def __iter__(self):
        return iter(self.columns)

    def __contains__(self, col):
        return col in self.columns

    def __len__(self):
        return self.size

    @property
    def size(self):
        return self._size

    @property
    def csize(self):
        try:
            return self._csize
        except AttributeError:
            self._csize = int(self.comm.allreduce(self.size))
            return self._csize

    # ---- column access
    def make_column(self, array):
        return array if isinstance(array, Column) else Column(array)

    def get_hardcolumn(self, col):
        f = find_column(self.__class__, col)
        if f is None:
            raise ValueError("no such column: %s" % col)
        return self.make_column(f(self))

    def __getitem__(self, sel):
        # a column
        if isinstance(sel, str):
            if sel in self._overrides:
                return self._overrides[sel]
            if sel in self.hardcolumns:
                return self.get_hardcolumn(sel)
            raise KeyError("column `%s` is not defined in this source; " % sel + "try adding column via `source[column] = data`")
        # a list of column names -> catalogue with those columns
        if isinstance(sel, (list, tuple)) and len(sel) and all(isinstance(s, str) for s in sel):
            missing = [s for s in sel if s not in self]
            if missing:
                raise KeyError("invalid column names: %s" % str(missing))
            return self._subset(slice(None), columns=list(sel))
        # boolean mask / slice / index array -> row subset
        return self._subset(sel)

    def _subset(self, index, columns=None):
        from ..source.catalog.array import ArrayCatalog
        if isinstance(index, Column):
            index = index.compute() if not isinstance(index, ConstantColumn) else index.materialize()
        names = columns if columns is not None else self.columns
        data = {}
        size = None
        for name in names:
            col = self[name]
            sub = col[index] if not (isinstance(index, slice) and index == slice(None)) else col
            data[name] = sub
            size = len(sub)
        out = ArrayCatalog.__new__(ArrayCatalog)
        CatalogSourceBase.__init__(out, self.comm)
        out._size = size if size is not None else 0
        out._csize = int(self.comm.allreduce(out._size))     # slicing is collective (as in the reference)
        out._overrides = {k: (v if isinstance(v, Column) else Column(v)) for k, v in data.items()}
        out.attrs.update(self.attrs)
        out.base = self
        return out

    def __setitem__(self, col, value):
        if not isinstance(col, str):
            raise ValueError("column names must be strings")
        if isinstance(value, Column):
            pass
        elif numpy.isscalar(value) or (isinstance(value, numpy.ndarray) and value.ndim == 0):
            value = ConstantColumn(value, self.size)
        else:
            value = Column(value)
        if len(value) != self.size:
            raise ValueError("error setting '%s' column, data must be array of size %d, not %d"
                             % (col, self.size, len(value)))
        self._overrides[col] = value

    def __delitem__(self, col):
        if col in self._overrides:
            del self._overrides[col]
        elif col in self.hardcolumns:
            raise ValueError("cannot delete a hard-coded column")
        else:
            raise KeyError("no such column %s" % col)

    def compute(self, *args, **kwargs):
        """materialise columns (reference: dask.compute, base/catalog.py:530-560)"""
        out = []
        for a in args:
            if isinstance(a, (list, tuple)):
                out.append([x.compute() if isinstance(x, Column) else x for x in a])
            else:
                out.append(a.compute() if isinstance(a, Column) else a)
        return out[0] if len(out) == 1 else tuple(out)

    def read(self, columns):
        """list of columns by name (base/catalog.py `read`)"""
        missing = set(columns) - set(self.columns)
        if len(missing) > 0:
            raise ValueError("source does not contain columns: %s; " % str(missing) +
                             "try adding columns via `source[column] = data`")
        return [self[col] for col in columns]

    def copy(self):
        return self._subset(slice(None))

    def view(self, type=None):
        return self.copy()

    # ---- mesh conversion (base/catalog.py:787-873)
    def to_mesh(self, Nmesh=None, BoxSize=None, dtype='f4', interlaced=False, compensated=False,
                resampler='cic', weight='Weight', value='Value', selection='Selection',
                position='Position', window=None):
        from ..source.mesh import CatalogMesh
        from ..pmesh.window import methods
        if window is not None:
            resampler = window
            import warnings
            warnings.warn("The window argument is deprecated. Use `resampler=` instead", DeprecationWarning, stacklevel=2)
        for col in [weight, selection]:
            if col not in self:
                raise ValueError("column '%s' missing; cannot create mesh" % col)
        if resampler not in methods:
            raise ValueError("valid resampler: %s" % str(list(methods)))
        if BoxSize is None:
            try:
                BoxSize = self.attrs['BoxSize']
            except KeyError:
                raise ValueError(("cannot convert particle source to a mesh; "
                                  "'BoxSize' keyword is not supplied and the CatalogSource "
                                  "does not define one in 'attrs'."))
        if Nmesh is None:
            try:
                Nmesh = self.attrs['Nmesh']
            except KeyError:
                raise ValueError(("cannot convert particle source to a mesh; "
                                  "'Nmesh' keyword is not supplied and the CatalogSource "
                                  "does not define one in 'attrs'."))
        return CatalogMesh(self, Nmesh=Nmesh, BoxSize=BoxSize, dtype=dtype,
                           Weight=self[weight], Selection=self[selection], Value=self[value],
                           Position=self[position], interlaced=interlaced, compensated=compensated,
                           resampler=resampler)


class _RowMover(object):
    """moves per-row tensors so that the row of global position rank[i] lands there, every rank keeping `n` rows: a
    gather on one rank, one all-to-all per column on several"""

    def __init__(self, comm, rank, n):
        self.comm = comm
        dev = rank.device
        if comm.size == 1:
            self.order = torch.empty(n, dtype=torch.int64, device=dev)
            self.order[rank] = torch.arange(n, dtype=torch.int64, device=dev)
            return
        sizes = comm.allgather(int(n))
        self.base = int(sum(sizes[:comm.rank]))
        bounds = torch.tensor(numpy.cumsum(sizes)[:-1].tolist(), dtype=torch.int64, device=dev)
        # rows in ascending destination position, hence grouped by destination rank
        self.by_pos = torch.argsort(rank)
        dest = torch.bucketize(rank.index_select(0, self.by_pos), bounds, right=True)
        self.sendcounts = torch.bincount(dest, minlength=comm.size).cpu().tolist()
        self.recvcounts = comm.alltoall_ints(self.sendcounts)
        self.at = self._send(rank) - self.base

    def _send(self, t):
        send = t.index_select(0, self.by_pos).contiguous()
        out = torch.empty((int(sum(self.recvcounts)),) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
        self.comm.all_to_all_single(out, send, list(self.recvcounts), list(self.sendcounts))
        return out

    def __call__(self, t):
        if self.comm.size == 1:
            return t.index_select(0, self.order.to(t.device))
        dev = self.at.device
        recv = self._send(t.to(dev))
        out = torch.empty_like(recv)
        out[self.at] = recv
        return out.to(t.device)


class CatalogSource(CatalogSourceBase):
    """a CatalogSourceBase with a fixed size and the default columns (base/catalog.py:876-1216)"""
    logger = logging.getLogger('CatalogSource')

    def __init__(self, comm):
        CatalogSourceBase.__init__(self, comm)
        if not hasattr(self, '_size'):
            raise ValueError("the `size` of the CatalogSource must be set before initializing the base class")
        # collective: every rank constructs the catalogue, so the global size is known from here on and
        # rank-0-only code (logging) may read `csize` without triggering a collective
        self._csize = int(self.comm.allreduce(self._size))

    def sort(self, keys, reverse=False, usecols=None):
        """
        Return a catalogue whose rows are sorted globally, across all ranks, by the input keys (base/catalog.py:1100).

        Rows are ordered lexicographically by `keys`, the first key primary, ascending (descending with `reverse`).
        Values compare numerically (the reference orders float keys by their bit patterns, which reverses negative
        values), and ties keep ascending global row order (the reference leaves them to mpsort).  Every rank keeps its
        number of rows, as the reference's in-place sort does.  The keys are sorted on the GPU; on several ranks every
        rank all-gathers the key columns, (8 K + 8) bytes per row of the whole catalogue for K keys
        (base/ordering.py), and the columns travel to their new ranks in one all-to-all each.

        Parameters
        ----------
        keys : str, list, tuple
            the names of the columns to sort by: integer or floating point, one-dimensional, without NaN
        reverse : bool, optional
            if ``True``, sort in descending order
        usecols : list, optional
            the names of the columns of the returned catalogue (default: all columns)
        """
        from .ordering import check_no_nan, global_rank, key_tensor
        from ..source.catalog.array import ArrayCatalog
        if isinstance(keys, str):
            keys = [keys]
        keys = list(keys)
        if len(set(keys)) != len(keys):
            raise ValueError("duplicated sort keys")
        bad = set(keys) - set(self.columns)
        if len(bad):
            raise ValueError("invalid sort keys: %s" % str(bad))
        if usecols is not None:
            if isinstance(usecols, str):
                usecols = [usecols]
            if not isinstance(usecols, (list, tuple)):
                raise ValueError("usecols should be a list or tuple of column names")
            bad = set(usecols) - set(self.columns)
            if len(bad):
                raise ValueError("invalid column names in usecols: %s" % str(bad))
        kt = [key_tensor(self[k], k) for k in keys]
        dev = torch.device("cuda", torch.cuda.current_device())
        kt = [k.to(dev) for k in kt]
        check_no_nan(self.comm, kt, keys)
        n = self.size
        rank = global_rank(self.comm, kt, n, dev, reverse=reverse)
        del kt
        names = self.columns if usecols is None else list(dict.fromkeys(usecols))
        move = _RowMover(self.comm, rank, n)
        data, const = {}, {}
        for name in names:
            col = self[name]
            if isinstance(col, ConstantColumn):
                const[name] = col.value
                continue
            a = col.compute()
            if _is_torch(a):
                data[name] = move(a)
            else:
                data[name] = move(torch.from_numpy(numpy.ascontiguousarray(a)).to(dev)).cpu().numpy()
        if not data:
            # only constant columns: the catalogue needs one array to know its size
            data = {name: numpy.full(n, value) for name, value in const.items()}
            const = {}
        out = ArrayCatalog(data, comm=self.comm, **self.attrs)
        for name, value in const.items():
            out[name] = ConstantColumn(value, n)
        return out

    @column(is_default=True)
    def Selection(self):
        """boolean selection column; True for every particle by default"""
        return ConstantColumn(True, self.size)

    @column(is_default=True)
    def Weight(self):
        """weight of each particle on the mesh; 1.0 by default"""
        return ConstantColumn(1.0, self.size)

    @column(is_default=True)
    def Value(self):
        """field value carried by each particle; 1.0 by default"""
        return ConstantColumn(1.0, self.size)
