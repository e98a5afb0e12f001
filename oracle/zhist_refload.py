"""
TEST INFRASTRUCTURE -- the reference's RedshiftHistogram, run verbatim on one rank.

Loads nbodykit/algorithms/zhist.py by file path and unmodified, on top of the stub package of oracle/refload.py, with a
stand-in for `transform.ConstantArray` (a NumPy array of one value instead of a dask array), `MPI.MAX`, and a minimal
source (`comm`, `size`, `compute`, `__contains__`, `__getitem__`).  Its `save` / `load` use the reference's own
JSONEncoder / JSONDecoder: nbodykit/utils.py is loaded verbatim as well, behind stand-ins for `mpsort`,
`astropy.units.Quantity` / `Unit` and `nbodykit.cosmology.Cosmology`.  scipy's spline is the real one.  Used by
tests/test_oracle_zhist_reference.py (pinning oracle/zhist_oracle.py) and tests/golden/make_zhist_golden.py (the
tests/golden/zhist_* fixtures).  The reference tree is absent on GPU machines: nothing that runs there may import this
module.
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

    def bcast(self, x, root=0):
        return x


def ConstantArray(value, size, chunks=100000):
    """transform.ConstantArray without dask: `size` copies of `value` (reference transform.py:89-106)"""
    ele = numpy.array(value)
    return numpy.lib.stride_tricks.as_strided(ele, [size] + list(ele.shape), [0] + list(ele.strides))


class Source(object):
    """the catalogue RedshiftHistogram reads: named NumPy columns"""

    def __init__(self, **columns):
        self.comm = Comm()
        self.columns = {k: numpy.asarray(v) for k, v in columns.items()}
        self.size = len(next(iter(self.columns.values()))) if self.columns else 0

    def __contains__(self, name):
        return name in self.columns

    def __getitem__(self, name):
        return self.columns[name]

    def compute(self, *args):
        out = tuple(numpy.asarray(a) for a in args)
        return out[0] if len(out) == 1 else out


class _Quantity(object):
    pass


class _RefCosmology(object):
    """what the reference's JSON coder needs of a Cosmology: `pars` and `from_dict`"""

    def __init__(self, pars):
        self.pars = dict(pars)

    @classmethod
    def from_dict(cls, pars):
        return cls(pars)


def load():
    """namespace with the reference's `RedshiftHistogram`, `scotts_bin_width` and JSON coder; idempotent"""
    if _ns:
        return _ns["ns"]
    refload.load()
    sys.modules["mpi4py"].MPI.MAX = "max"
    sys.modules["mpi4py.MPI"].MAX = "max"
    if "mpsort" not in sys.modules:
        refload._stub("mpsort")
    for name in ("astropy", "astropy.units"):
        if name not in sys.modules:
            refload._stub(name)
    sys.modules["astropy.units"].Quantity = getattr(sys.modules["astropy.units"], "Quantity", _Quantity)
    sys.modules["astropy.units"].Unit = getattr(sys.modules["astropy.units"], "Unit", str)
    cosmo = sys.modules.get("nbodykit.cosmology") or refload._stub("nbodykit.cosmology")
    if not hasattr(cosmo, "Cosmology"):
        cosmo.Cosmology = _RefCosmology
    utils = refload._load("nbodykit._zhist_ref_utils", "nbodykit/utils.py")
    stub_utils = sys.modules["nbodykit.utils"]
    stub_utils.JSONEncoder = utils.JSONEncoder
    stub_utils.JSONDecoder = utils.JSONDecoder
    transform = sys.modules.get("nbodykit.transform") or refload._stub("nbodykit.transform")
    transform.ConstantArray = ConstantArray
    mod = refload._load("nbodykit.algorithms.zhist", "nbodykit/algorithms/zhist.py")
    ns = types.SimpleNamespace(module=mod, RedshiftHistogram=mod.RedshiftHistogram, scotts_bin_width=mod.scotts_bin_width,
                               JSONEncoder=utils.JSONEncoder, JSONDecoder=utils.JSONDecoder, Source=Source, Comm=Comm)
    _ns["ns"] = ns
    return ns


def run(z, fsky, cosmo, bins=None, w=None):
    """the reference's RedshiftHistogram of one rank's redshifts z (and weights w)"""
    ns = load()
    cols = dict(z=z)
    if w is not None:
        cols['w'] = w
    return ns.RedshiftHistogram(Source(**cols), fsky, cosmo, bins=bins, redshift='z', weight='w' if w is not None else None)


def load_saved(path):
    """the reference's RedshiftHistogram.load of a file"""
    return load().RedshiftHistogram.load(path, comm=Comm())


def available():
    return refload.available()


class CosmoDict(dict):
    """a cosmology the reference accepts: its `attrs['cosmo'] = dict(cosmo)` needs a mapping, its volumes
    `comoving_distance`"""

    def __init__(self, cosmo):
        dict.__init__(self, cosmo.pars)
        self._cosmo = cosmo

    def comoving_distance(self, z):
        return self._cosmo.comoving_distance(z)
