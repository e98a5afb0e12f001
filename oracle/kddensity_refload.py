"""
TEST INFRASTRUCTURE -- the reference's KDDensity, run verbatim on one rank.

Loads nbodykit/algorithms/kdtree.py by file path and unmodified, on top of the stub package of oracle/refload.py, with
single-rank stand-ins for what `KDDensity.run` calls: `split_size_3d`, an identity `GridND` domain whose layout exchanges
nothing and whose `gather(mode=fmin)` returns its input, and a minimal source (`comm`, `attrs`, `csize`, `compute`,
`__contains__`, `__getitem__`).  scipy's cKDTree is the real one.  Used by tests/test_oracle_kddensity_reference.py
(pinning oracle/kddensity_oracle.py) and tests/golden/make_kddensity_golden.py (the tests/golden/kddensity_*.npz
fixtures).  The reference tree is absent on GPU machines: nothing that runs there may import this module.
"""
import sys
import types

import numpy

from . import refload

_ns = {}


class Comm(object):
    rank = 0
    size = 1

    def allreduce(self, x, op=None):
        return x


class _Layout(object):
    def exchange(self, x):
        return numpy.array(x, copy=True)

    def gather(self, x, mode=None):
        return x


class GridND(object):
    def __init__(self, comm=None, periodic=True, edges=None, **kw):
        self.edges = edges

    def decompose(self, pos, smoothing=0):
        return _Layout()


def split_size_3d(s):
    return [1, 1, 1] if s == 1 else None


class Source(object):
    """the catalogue KDDensity reads"""

    def __init__(self, pos, BoxSize):
        self.comm = Comm()
        self.attrs = {'BoxSize': BoxSize}
        self.pos = numpy.asarray(pos)
        self.csize = len(self.pos)

    def __contains__(self, name):
        return name == 'Position'

    def __getitem__(self, name):
        return self.pos

    def compute(self, x):
        return x


def load():
    """the reference's `KDDensity` class; idempotent"""
    if _ns:
        return _ns["ns"]
    refload.load()
    sys.modules["nbodykit.utils"].split_size_3d = split_size_3d
    domain = refload._stub("pmesh.domain", GridND=GridND)
    sys.modules["pmesh"].domain = domain
    mod = refload._load("nbodykit.algorithms.kdtree", "nbodykit/algorithms/kdtree.py")
    ns = types.SimpleNamespace(module=mod, KDDensity=mod.KDDensity, Source=Source)
    _ns["ns"] = ns
    return ns


def run(pos, BoxSize):
    """(density, attrs) of the reference's KDDensity on `pos`"""
    ns = load()
    r = ns.KDDensity(Source(pos, BoxSize))
    return numpy.asarray(r.density), r.attrs


def available():
    return refload.available()
