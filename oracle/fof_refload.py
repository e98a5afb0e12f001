"""
TEST INFRASTRUCTURE -- the reference's friends-of-friends helpers, loaded verbatim.

Loads nbodykit/algorithms/fof.py by file path and unmodified, on top of the stub package of oracle/refload.py, with
single-rank stand-ins for what it imports: `mpsort.sort`, `nbodykit.utils.DistributedArray` / `ScatterArray` /
`split_size_3d`, `nbodykit.source.catalog.ArrayCatalog`, and an MPI communicator with `Allreduce`.  Exposes
`_assign_labels`, `centerofmass`, `count`, `equiv_class` and `fof_catalog`.  Used by tests/test_oracle_fof_reference.py
(pinning oracle/fof_oracle.py) and tests/golden/make_fof_golden.py (the tests/golden/fof_*.npz fixtures).  The reference
tree is absent on GPU machines: nothing that runs there may import this module.
"""
import sys
import types

import numpy

from . import refload

_ns = {}


class Comm(object):
    """single-rank communicator with the buffer collectives fof.py calls"""
    rank = 0
    size = 1

    def allgather(self, x):
        return [x]

    def allreduce(self, x, op=None):
        return x

    def Allreduce(self, sendbuf, recvbuf, op=None):
        pass

    def bcast(self, x, root=0):
        return x

    def barrier(self):
        pass


class DistributedArray(object):
    """one-rank DistributedArray (reference utils.py:534-762): on a single rank `sort` is a local sort,
    `unique_labels` is numpy.unique's inverse and `bincount` a plain bincount"""

    def __init__(self, local, comm):
        self.local = local
        self.comm = comm

    def sort(self, orderby=None):
        _mpsort_sort(self.local, orderby)

    def __getitem__(self, key):
        return DistributedArray(self.local[key], self.comm)

    def unique_labels(self):
        _, label = numpy.unique(self.local, return_inverse=True)
        return DistributedArray(numpy.int64(label).reshape(-1), self.comm)

    def bincount(self, weights=None, local=False, shared_edges=True):
        N = numpy.bincount(self.local, weights)
        return N if local else DistributedArray(N, self.comm)


def _mpsort_sort(data, orderby=None, comm=None):
    """mpsort.sort on one rank: sort the structured array in place by one field"""
    arg = numpy.argsort(data[orderby], kind="stable")
    data[...] = data[arg]


def _scatter_array(data, comm, root=0, counts=None):
    return data


class Source(object):
    """the parts of a CatalogSource fof_catalog reads: columns, `compute`, `attrs`"""

    class _Col(object):
        def __init__(self, a):
            self.a = a

        def compute(self):
            return self.a

    def __init__(self, columns, **attrs):
        self.columns = columns
        self.attrs = attrs

    def __contains__(self, name):
        return name in self.columns

    def __getitem__(self, name):
        return Source._Col(self.columns[name])

    def compute(self, col):
        return col.compute()


def load():
    """namespace with the reference's fof.py helpers; idempotent"""
    if _ns:
        return _ns["ns"]
    refload.load()                                     # the stub nbodykit package (raises when the tree is absent)
    _mpsort = types.ModuleType("mpsort")
    _mpsort.sort = _mpsort_sort
    sys.modules["mpsort"] = _mpsort
    utils = sys.modules["nbodykit.utils"]
    utils.DistributedArray = DistributedArray
    utils.ScatterArray = _scatter_array
    utils.split_size_3d = lambda s: numpy.array([1, 1, s])
    refload._stub("nbodykit.source.catalog", ArrayCatalog=object)
    mod = refload._load("nbodykit.algorithms.fof", "nbodykit/algorithms/fof.py")
    # the MPI names fof.py uses at call time, beyond those of refload's stub
    mod.MPI.IN_PLACE = None
    mod.MPI.MAX = "max"
    ns = types.SimpleNamespace(module=mod, Comm=Comm, Source=Source, _assign_labels=mod._assign_labels,
                               centerofmass=mod.centerofmass, count=mod.count, equiv_class=mod.equiv_class,
                               fof_catalog=mod.fof_catalog)
    _ns["ns"] = ns
    return ns


def available():
    return refload.available()
