"""
TEST INFRASTRUCTURE -- the reference's cylinder-grouping code, run verbatim on one rank.

Loads nbodykit/algorithms/cgm.py by file path and unmodified, on top of the stub package of oracle/refload.py, with
single-rank stand-ins for what `cgm()` calls: a kdcount `KDTree(...).root.enum` built on scipy's cKDTree (self-pairs
included, pairs at distance <= rmax), an identity `GridND` domain whose layouts exchange and gather nothing, a
stable-argsort `mpsort.sort`, and the communicator.  Also extracts `direct_cgm` from the reference's test_cgm.py with
`ast`.  Used by tests/test_oracle_cgm_reference.py (pinning oracle/cgm_oracle.py) and tests/golden/make_cgm_golden.py
(the tests/golden/cgm_*.npz fixtures).  The reference tree is absent on GPU machines: nothing that runs there may
import this module.
"""
import ast
import os
import sys
import types

import numpy
from scipy.spatial import cKDTree

from . import refload

_ns = {}


class Comm(object):
    rank = 0
    size = 1

    def allgather(self, x):
        return [x]

    def allreduce(self, x, op=None):
        return x

    def gather(self, x, root=0):
        return [x]

    def bcast(self, x, root=0):
        return x


class _Node(object):
    def __init__(self, pos, boxsize):
        self.pos = numpy.asarray(pos, dtype='f8')
        self.boxsize = None if boxsize is None else numpy.asarray(boxsize, dtype='f8')

    def enum(self, other, rmax, process):
        """every pair (i of self, j of other) within rmax, self-pairs included, in one callback"""
        t1 = cKDTree(self.pos, boxsize=self.boxsize)
        t2 = cKDTree(other.pos, boxsize=other.boxsize)
        lists = t1.query_ball_tree(t2, rmax)
        i = numpy.repeat(numpy.arange(len(lists)), [len(l) for l in lists]).astype('i8')
        j = numpy.concatenate([numpy.asarray(l, dtype='i8') for l in lists]) if len(lists) else numpy.zeros(0, 'i8')
        process(None, i, j)


class KDTree(object):
    def __init__(self, pos, boxsize=None):
        self.root = _Node(pos, boxsize)


class _Layout(object):
    def exchange(self, x):
        return x

    def gather(self, x, mode=None):
        return x


class GridND(object):
    def __init__(self, grid, comm=None):
        self.grid = grid

    def decompose(self, pos, smoothing=0):
        return _Layout()


def _mpsort_sort(data, orderby=None, comm=None):
    arg = numpy.argsort(data[orderby], kind="stable")
    data[...] = data[arg]


class Data(object):
    """the sorted catalogue `cgm()` reads: columns, `compute`, `len`"""

    def __init__(self, **cols):
        self.cols = cols

    def __getitem__(self, name):
        return self.cols[name]

    def __len__(self):
        return len(self.cols['Position'])

    def compute(self, *cols):
        return cols


def load():
    """namespace with the reference's `cgm` and `direct_cgm`; idempotent"""
    if _ns:
        return _ns["ns"]
    refload.load()
    refload._stub("kdcount", KDTree=KDTree)
    refload._stub("mpsort", sort=_mpsort_sort)
    domain = refload._stub("pmesh.domain", GridND=GridND)
    sys.modules["pmesh"].domain = domain
    if "nbodykit.source.catalog" not in sys.modules:
        refload._stub("nbodykit.source.catalog", ArrayCatalog=object)
    mod = refload._load("nbodykit.algorithms.cgm", "nbodykit/algorithms/cgm.py")
    src = open(os.path.join(refload.REF, "nbodykit", "algorithms", "tests", "test_cgm.py")).read()
    fn = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == "direct_cgm"][0]
    g = {"numpy": numpy}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), "test_cgm.py", "exec"), g)
    ns = types.SimpleNamespace(module=mod, cgm=mod.cgm, direct_cgm=g["direct_cgm"], Comm=Comm, Data=Data,
                               GridND=GridND)
    _ns["ns"] = ns
    return ns


def run_cgm(pos, prio, rperp, rpar, los, boxsize):
    """the reference's cgm() on rows already ranked by `prio` (0 .. N-1, larger first): (cgm_type, cgm_haloid,
    num_cgm_sats) in the input row order"""
    ns = load()
    n = len(pos)
    order = numpy.argsort(prio, kind="stable")
    data = Data(Position=numpy.asarray(pos)[order], origind=order.astype('u4'),
                sortindex=numpy.arange(n, dtype='i8'))
    out = ns.cgm(Comm(), data, GridND(None), rperp, rpar, los, boxsize)
    return (numpy.asarray(out['cgm_type']), numpy.asarray(out['cgm_haloid']), numpy.asarray(out['num_cgm_sats']))


def available():
    return refload.available()
