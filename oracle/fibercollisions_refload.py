"""
TEST INFRASTRUCTURE -- the reference's FiberCollisions, run verbatim on one rank.

Loads nbodykit/algorithms/fibercollisions.py by file path and unmodified, on top of the stub package of
oracle/refload.py, with single-rank stand-ins for what it calls: `FOF` from oracle/fof_oracle.py (periodic box 2.2,
labels by size then smallest row), a stable-argsort `mpsort.sort`, astropy's `NumpyRNGContext` (seed NumPy's global
generator, restore it afterwards), a NumPy `SkyToUnitSphere` and a minimal `ArrayCatalog`.  Used by
tests/test_oracle_fibercollisions_reference.py (pinning oracle/fibercollisions_oracle.py) and
tests/golden/make_fibercollisions_golden.py (the tests/golden/fibercollisions_*.npz fixtures).  The reference tree is
absent on GPU machines: nothing that runs there may import this module.
"""
import sys
import types

import numpy

from . import refload

_ns = {}


class Comm(object):
    rank = 0
    size = 1

    def allgather(self, x):
        return [x]

    def allreduce(self, x, op=None):
        return x

    def bcast(self, x, root=0):
        return x


class _Lazy(numpy.ndarray):
    """an array with the `compute()` of a dask array"""

    def compute(self):
        return numpy.ascontiguousarray(numpy.asarray(self))


def SkyToUnitSphere(ra, dec, degrees=True, frame='icrs'):
    ra, dec = numpy.broadcast_arrays(numpy.asarray(ra), numpy.asarray(dec))
    if degrees:
        ra, dec = numpy.deg2rad(ra), numpy.deg2rad(dec)
    return numpy.vstack([numpy.cos(dec) * numpy.cos(ra), numpy.cos(dec) * numpy.sin(ra), numpy.sin(dec)]).T.view(_Lazy)


class ArrayCatalog(object):
    def __init__(self, data, comm=None, **attrs):
        self.data = data
        self.comm = comm if comm is not None else Comm()
        self.attrs = dict(attrs)

    @staticmethod
    def make_column(x):
        return numpy.asarray(x)

    def __getitem__(self, name):
        return self.data[name]

    def compute(self, x):
        return x


class FOF(object):
    def __init__(self, source, linking_length, nmin, absolute=False):
        from . import fof_oracle
        assert absolute
        pos = source['Position']
        self.labels = fof_oracle.fof_labels(pos, linking_length, nmin, box=source.attrs['BoxSize']).astype('i4')


class NumpyRNGContext(object):
    def __init__(self, seed):
        self.seed = seed

    def __enter__(self):
        self.state = numpy.random.get_state()
        numpy.random.seed(self.seed)

    def __exit__(self, *exc):
        numpy.random.set_state(self.state)


def _mpsort_sort(data, orderby=None, out=None, comm=None):
    arg = numpy.argsort(data[orderby], kind="stable")
    out[...] = data[arg]


def load():
    """the reference's `FiberCollisions` class; idempotent"""
    if _ns:
        return _ns["ns"]
    refload.load()
    sys.modules["mpi4py"].MPI.MAX = "max"
    refload._stub("mpsort", sort=_mpsort_sort)
    refload._stub("astropy")
    refload._stub("astropy.utils")
    refload._stub("astropy.utils.misc", NumpyRNGContext=NumpyRNGContext)
    for name, attrs in (("nbodykit.source.catalog", dict(ArrayCatalog=ArrayCatalog)),
                        ("nbodykit.transform", dict(SkyToUnitSphere=SkyToUnitSphere)),
                        ("nbodykit.algorithms", dict(FOF=FOF))):
        mod = sys.modules.get(name) or refload._stub(name)
        mod.__dict__.update(attrs)
    mod = refload._load("nbodykit.algorithms.fibercollisions", "nbodykit/algorithms/fibercollisions.py")
    ns = types.SimpleNamespace(module=mod, FiberCollisions=mod.FiberCollisions)
    _ns["ns"] = ns
    return ns


def run(ra, dec, collision_radius=62 / 60. / 60., seed=42, degrees=True):
    """(pos, Label, Collided, NeighborID, rad) of the reference's FiberCollisions on one rank"""
    ns = load()
    r = ns.FiberCollisions(numpy.asarray(ra), numpy.asarray(dec), collision_radius=collision_radius, seed=seed,
                           degrees=degrees, comm=Comm())
    lab = r.labels.data
    pos = numpy.asarray(r.source['Position'])
    return (pos, numpy.asarray(lab['Label']), numpy.asarray(lab['Collided']), numpy.asarray(lab['NeighborID']),
            r._collision_radius_rad)


def available():
    return refload.available()
