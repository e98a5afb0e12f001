"""
HaloCatalog and PopulatedHaloCatalog (API of nbodykit/source/catalog/halos.py) on one or several GPUs.

The reference hands each rank's halos to halotools on the CPU.  Here the Zheng07, Leauthaud11 and Hearin15 models of
:mod:`nbodykit_b200.hod` are evaluated by this package's kernels (csrc/hod.cu) to the contract of DESIGN.md 4.13: one
occupation draw per halo, a scan for the galaxy rows, then one thread per galaxy for its position and velocity.
Hearin15 also ranks each halo's secondary property among the halos of its mass bin on all ranks, once per catalogue.
Every draw is a counter-based hash of (seed, stream, global halo row, draw index), so the catalogue is the same for any
number of ranks and any split of the halo rows.  Galaxies stay on the rank of their halo: on every rank the centrals
of its halos come first, in halo order, then the satellites, in (halo, satellite) order.
"""
import logging
import math
import numbers

import numpy
import torch

from ... import CurrentMPIComm
from ... import transform
from ..._lib import F4, F8, check, darr, lib, stage
from ...base.catalog import CatalogSource, CatalogSourceBase, Column, ConstantColumn, column
from ...base.ordering import global_rank, key_tensor
from ...cosmology import Cosmology, G_KMS2_MPC_PER_MSUN
from ...pmesh.pm import _ptr, _stream, as_device_tensor, current_device
from .array import ArrayCatalog

__all__ = ['HaloCatalog', 'PopulatedHaloCatalog']


def _check_cosmo(cosmo, what):
    if not isinstance(cosmo, Cosmology):
        raise NotImplementedError("%s: a cosmology other than nbodykit_b200's Cosmology is handed to halotools by the "
                                  "reference; halotools is not a dependency of nbodykit_b200" % what)


class HaloCatalog(CatalogSource):
    r"""
    A catalogue of halos, which can be populated with galaxies by :meth:`populate`.

    Parameters
    ----------
    source : CatalogSource
        the source holding the halos
    cosmo : :class:`~nbodykit_b200.cosmology.Cosmology`
        the cosmology
    redshift : float
        the redshift of the halos
    mdef : str, optional
        the mass definition of ``Mass``, for the default ``Radius`` and ``Concentration``: ``'vir'``, ``'XXXc'`` or
        ``'XXXm'`` with XXX an integer overdensity
    mass, position, velocity : str, optional
        the column names of the mass (M_sun/h), position (Mpc/h) and velocity (km/s) in ``source``
    """
    logger = logging.getLogger("HaloCatalog")

    def __init__(self, source, cosmo, redshift, mdef='vir', mass='Mass', position='Position', velocity='Velocity'):
        required = ['mass', 'position', 'velocity']
        for name, col in zip(required, [mass, position, velocity]):
            if col is None:
                raise ValueError("the %s column cannot be None in HaloCatalog" % name)
        if not isinstance(source, CatalogSourceBase):
            raise TypeError("input source to HaloCatalog should be a CatalogSource")
        for name, col in zip(required, [mass, position, velocity]):
            if col not in source:
                raise ValueError("input source is missing the %s column; '%s' does not exist" % (name, col))
        _check_cosmo(cosmo, "HaloCatalog")
        redshift = float(redshift)
        if not (math.isfinite(redshift) and redshift > -1):
            raise ValueError("HaloCatalog: the redshift must be finite and above -1 (got %r)" % redshift)
        transform._threshold(cosmo, torch.tensor(redshift, dtype=torch.float64), mdef)   # ValueError for a bad mdef

        self._source = source
        self.cosmo = cosmo
        self.attrs.update(source.attrs)
        self.attrs['redshift'] = redshift
        self.attrs['cosmo'] = dict(cosmo.pars)
        self.attrs['mass'] = mass
        self.attrs['velocity'] = velocity
        self.attrs['position'] = position
        self.attrs['mdef'] = mdef
        self.attrs['halo_mass_key'] = 'halo_m' + mdef
        self.attrs['halo_radius_key'] = 'halo_r' + mdef
        self._size = source.size
        CatalogSource.__init__(self, comm=source.comm)

    @column
    def Mass(self):
        """the halo mass, in M_sun/h"""
        return self._source[self.attrs['mass']]

    @column
    def Position(self):
        """the halo position, in Mpc/h"""
        return self._source[self.attrs['position']]

    @column
    def Velocity(self):
        """the halo velocity, in km/s"""
        return self._source[self.attrs['velocity']]

    @column
    def VelocityOffset(self):
        """the redshift-space offset of the velocity in Mpc/h: ``Velocity`` times (1 + z) / (100 E(z))"""
        z = self.attrs['redshift']
        return self['Velocity'] * ((1 + z) / (100. * self.cosmo.efunc(z)))

    @column
    def Concentration(self):
        """the NFW concentration, :func:`~nbodykit_b200.transform.HaloConcentration` (Dutton & Maccio 2014).  Overwrite
        this column to use another mass-concentration relation"""
        return transform.HaloConcentration(self['Mass'], self.cosmo, self.attrs['redshift'], mdef=self.attrs['mdef'])

    @column
    def Radius(self):
        """the proper halo radius in Mpc/h, :func:`~nbodykit_b200.transform.HaloRadius`"""
        return transform.HaloRadius(self['Mass'], self.cosmo, self.attrs['redshift'], mdef=self.attrs['mdef'])

    def to_halotools(self, BoxSize=None):
        """the reference's halotools catalogue; halotools is not a dependency of this package"""
        raise NotImplementedError("HaloCatalog.to_halotools needs halotools, which is not a dependency of "
                                  "nbodykit_b200; use populate() to populate the halos on the GPU")

    def populate(self, model, BoxSize=None, seed=None, **params):
        """
        Populate the halos with galaxies of an HOD ``model`` on the GPU (DESIGN.md 4.13).

        Parameters
        ----------
        model : :class:`~nbodykit_b200.hod.Zheng07Model`, :class:`~nbodykit_b200.hod.Leauthaud11Model` or
            :class:`~nbodykit_b200.hod.Hearin15Model`, class or instance
            the occupation model
        BoxSize : float, 3-vector, optional
            the box the galaxy positions wrap into; ``attrs['BoxSize']`` when not given
        seed : int, optional
            the seed of the draws, in [0, 2^32); rank 0 draws one when None
        **params :
            model parameters

        Returns
        -------
        :class:`PopulatedHaloCatalog`
        """
        model = _as_model(model)
        model.update(params)
        model.check()
        box = _box(BoxSize if BoxSize is not None else self.attrs.get('BoxSize', None))
        seed = _seed(self.comm, seed)
        occ = _occupation(model, self.attrs['redshift'])
        sec = _check_sec(self, model)
        halos = _Halos(self, box, sec)
        return PopulatedHaloCatalog._populate(halos, model, seed, self.cosmo, self.comm, occ)


def _as_model(model):
    from ...hod import HODModel, Hearin15Model, Leauthaud11Model, Zheng07Model
    if isinstance(model, type) and issubclass(model, HODModel):
        model = model()
    if not isinstance(model, HODModel):
        raise TypeError("model for populating mocks should be an nbodykit_b200.hod.HODModel subclass (got %r)" % (model,))
    for cls in (Hearin15Model, Leauthaud11Model, Zheng07Model):
        if isinstance(model, cls):
            # a private copy: populate and repopulate update its parameters
            return cls(**dict(model.arguments(), **model.param_dict))
    raise NotImplementedError("only Zheng07Model, Leauthaud11Model and Hearin15Model are implemented (got %s)"
                              % type(model).__name__)


def _occupation(model, redshift):
    """the host-side inputs of the occupation kernel (the SMHM spline of Leauthaud11 and Hearin15; None for Zheng07)"""
    from ...hod import Leauthaud11Model
    return model.occupation(redshift) if isinstance(model, Leauthaud11Model) else None


def _check_sec(cat, model):
    """the name of the Hearin15 secondary halo property (None for other models), after checking on all ranks that it is
    a 1-D column of finite numbers"""
    from ...hod import Hearin15Model
    if not isinstance(model, Hearin15Model):
        return None
    name = model.sec_haloprop
    if name not in cat:
        raise ValueError("Hearin15Model: the halo catalogue has no sec_haloprop column '%s'" % name)
    v = _values(cat[name])
    shape = tuple(v.shape)
    if isinstance(v, torch.Tensor):
        nonfinite = int((~torch.isfinite(v)).sum().item()) if (v.is_floating_point() or v.is_complex()) else 0
        numeric = v.is_floating_point() or v.dtype in (torch.int8, torch.uint8, torch.int16, torch.int32, torch.int64)
    else:
        v = numpy.asarray(v)
        numeric = numpy.issubdtype(v.dtype, numpy.integer) or numpy.issubdtype(v.dtype, numpy.floating)
        nonfinite = int((~numpy.isfinite(v)).sum()) if numeric else 0
    bad_shape = int(_allreduce(cat.comm, int(len(shape) != 1 or not numeric)))
    nonfinite = int(_allreduce(cat.comm, nonfinite))
    if bad_shape:
        raise ValueError("Hearin15Model: sec_haloprop '%s' must be a one-dimensional numeric column" % name)
    if nonfinite:
        raise ValueError("Hearin15Model: sec_haloprop '%s' has %d non-finite values" % (name, nonfinite))
    return name


def _allreduce(comm, x):
    """the sum of x over the ranks"""
    return comm.allreduce(x) if comm.size > 1 else x


def _box(BoxSize):
    if BoxSize is None:
        raise ValueError("please specify a 'BoxSize' to populate the halos (none in the attrs either)")
    L = numpy.broadcast_to(numpy.asarray(BoxSize, dtype='f8').reshape(-1), (3,)).copy() \
        if numpy.size(BoxSize) in (1, 3) else None
    if L is None or not (numpy.isfinite(L).all() and (L > 0).all()):
        raise ValueError("BoxSize must be one or three finite positive numbers (got %r)" % (BoxSize,))
    return L


def _seed(comm, seed):
    if seed is None:
        seed = int(numpy.random.default_rng().integers(0, 1 << 32)) if comm.rank == 0 else None
        return int(comm.bcast(seed, root=0))
    if isinstance(seed, (bool, numpy.bool_)) or not isinstance(seed, numbers.Integral) or not 0 <= int(seed) < (1 << 32):
        raise ValueError("seed must be an integer in [0, 2^32) (got %r)" % (seed,))
    return int(seed)


def _values(col):
    if isinstance(col, ConstantColumn):
        col = col.materialize()
    return col.compute() if isinstance(col, Column) else col


class _Halos(object):
    """the halo columns the kernels read, on the device, and this rank's first global halo row; for Hearin15 the
    secondary halo property `sec` and the percentiles of each halo in its mass bin, cached per (sec, bin width)"""

    def __init__(self, cat, box, sec=None):
        comm = cat.comm
        self.comm = comm
        cols = {k: _values(cat[k]) for k in ('Mass', 'Radius', 'Concentration', 'Position', 'Velocity')}
        bad = 0
        for k in ('Mass', 'Radius', 'Concentration'):
            v = cols[k]
            if isinstance(v, torch.Tensor):
                bad += int((~(torch.isfinite(v) & (v > 0))).sum().item())
            else:
                v = numpy.asarray(v)
                bad += int((~(numpy.isfinite(v) & (v > 0))).sum())
        for k in ('Position', 'Velocity'):
            if tuple(cols[k].shape[1:]) != (3,):
                bad += 1
        bad = int(comm.allreduce(bad))
        if bad:
            raise ValueError("populate: %d halos have a non-finite or non-positive Mass, Radius or Concentration, or "
                             "Position / Velocity are not (N, 3)" % bad)
        n = int(cat.size)
        if n >= (1 << 30):
            raise ValueError("populate: at most 2^30 - 1 halos per rank (got %d)" % n)
        sizes = comm.allgather(n)
        if sum(sizes) == 0:
            raise ValueError("no particles in catalog after populating halo catalog: there are no halos")
        self.n, self.h0 = n, int(sum(sizes[:comm.rank]))
        dev = current_device()
        pos = as_device_tensor(cols['Position'], device=dev)
        if pos.dtype not in (torch.float32, torch.float64):
            pos = pos.to(torch.float64)
        self.pos = pos.reshape(n, 3).contiguous()
        self.vel = as_device_tensor(cols['Velocity'], dtype=self.pos.dtype, device=dev).reshape(n, 3).contiguous()
        f8 = torch.float64
        self.mass = as_device_tensor(cols['Mass'], dtype=f8, device=dev).reshape(n).contiguous()
        self.radius = as_device_tensor(cols['Radius'], dtype=f8, device=dev).reshape(n).contiguous()
        self.conc = as_device_tensor(cols['Concentration'], dtype=f8, device=dev).reshape(n).contiguous()
        self.box = box
        self.attrs = dict(cat.attrs)
        self.attrs['BoxSize'] = box.copy()
        z = cat.attrs['redshift']
        self.rsd = (1 + z) / (100. * cat.cosmo.efunc(z))
        from ...hod import jeans_table
        self.table = torch.from_numpy(jeans_table()).to(dev)
        self.sec = {}
        if sec is not None:
            self.sec[sec] = key_tensor(cat[sec], sec, device=dev)
        self._pct = {}

    def percentiles(self, sec, d):
        """float64 (n,): (rank + 1) / N_bin of each halo among the N_bin halos of all ranks in its mass bin
        floor(log10 M / d), ranked by (sec, global row)"""
        key = (sec, d)
        if key not in self._pct:
            comm, n = self.comm, self.n
            with stage("hod_percentile"):
                b = torch.floor(torch.log10(self.mass) / d)
                lo = float(b.min().item()) if n else math.inf
                hi = float(b.max().item()) if n else -math.inf
                if comm.size > 1:
                    lo, hi = float(comm.allreduce(lo, "min")), float(comm.allreduce(hi, "max"))
                nb = hi - lo + 1
                if not nb <= (1 << 24):
                    raise ValueError("Hearin15Model: %g mass bins of width dlog10_prim_haloprop = %r; at most 2^24"
                                     % (nb, d))
                bins = (b - lo).to(torch.int64)
                pos = global_rank(comm, [bins, self.sec[sec]], n, self.mass.device)
                cnt = torch.bincount(bins, minlength=int(nb)) if n else \
                    torch.zeros(int(nb), dtype=torch.int64, device=self.mass.device)
                if comm.size > 1:
                    comm.allreduce_tensor(cnt, "sum")
                start = torch.cumsum(cnt, 0) - cnt
                self._pct[key] = ((pos - start[bins] + 1).to(torch.float64) / cnt[bins].to(torch.float64)).contiguous()
        return self._pct[key]

    def run(self, model, seed, occ=None):
        """the galaxy columns of (model, seed) on this rank, and the local numbers of centrals and galaxies; `occ` holds
        the host-side inputs of the SMHM occupation (Leauthaud11, Hearin15)"""
        from ...hod import JEANS_HS, JEANS_K, JEANS_S0, Hearin15Model
        n, dev = self.n, self.pos.device
        p = model.param_dict
        L = lib()
        counts = torch.empty(2 * n, dtype=torch.int64, device=dev)
        if occ is None:
            with stage("hod_occupy"):
                check(L.nbk_hod_occupy(_ptr(self.mass), F8, n, self.h0, p['logMmin'], p['sigma_logM'],
                                       10. ** p['logM0'], 10. ** p['logM1'], p['alpha'],
                                       int(model.modulate_with_cenocc), seed, _ptr(counts), _stream()),
                      "nbk_hod_occupy")
        else:
            pct, split, acen, asat = None, 0.5, 0.0, 0.0
            if isinstance(model, Hearin15Model):
                pct = self.percentiles(model.sec_haloprop, model.dlog10_prim_haloprop)
                split = model.split
                acen, asat = model.strengths()
            tc = torch.from_numpy(numpy.concatenate([occ['t'], occ['c']])).to(dev)
            nt = occ['t'].size
            with stage("hod_occupy"):
                check(L.nbk_hod_occupy_smhm(_ptr(self.mass), F8, n, self.h0, _ptr(tc), nt, _ptr(tc[nt:]),
                                            model.threshold, p['scatter_model_param1'], occ['Msat'], occ['Mcut'],
                                            p['alphasat'], int(model.modulate_with_cenocc),
                                            _ptr(pct), split, acen, asat, seed,
                                            _ptr(counts), _stream()), "nbk_hod_occupy_smhm")
        with stage("hod_scan"):
            offsets = torch.empty(2 * n + 1, dtype=torch.int64, device=dev)
            wb = int(L.nbk_hod_scan_workspace(2 * n))
            if wb < 0:
                raise RuntimeError("nbk_hod_scan_workspace failed for %d counts" % (2 * n))
            work = torch.empty(max(wb, 1), dtype=torch.uint8, device=dev)
            check(L.nbk_hod_scan(_ptr(counts), 2 * n, _ptr(offsets), _ptr(work), wb, _stream()), "nbk_hod_scan")
            ends = offsets[[n, 2 * n]].cpu()
        ncen, ngal = int(ends[0]), int(ends[1])
        T = self.pos.dtype
        pos = torch.empty((ngal, 3), dtype=T, device=dev)
        vel = torch.empty((ngal, 3), dtype=T, device=dev)
        voff = torch.empty((ngal, 3), dtype=T, device=dev)
        hcd = torch.empty(ngal, dtype=torch.float64, device=dev)
        gal_type = torch.empty(ngal, dtype=torch.int32, device=dev)
        halo_id = torch.empty(ngal, dtype=torch.int64, device=dev)
        with stage("hod_emit"):
            check(L.nbk_hod_emit(_ptr(offsets), n, ngal, self.h0, _ptr(self.pos), _ptr(self.vel),
                                 F4 if T == torch.float32 else F8, _ptr(self.mass), _ptr(self.radius), _ptr(self.conc),
                                 darr(self.box), G_KMS2_MPC_PER_MSUN, float(self.rsd), _ptr(self.table), JEANS_K,
                                 JEANS_S0, JEANS_HS, seed, _ptr(pos), _ptr(vel), _ptr(voff), _ptr(hcd), _ptr(gal_type),
                                 _ptr(halo_id), _stream()), "nbk_hod_emit")
        local = halo_id - self.h0
        mdef = self.attrs['mdef']
        data = {'Position': pos, 'Velocity': vel, 'VelocityOffset': voff, 'gal_type': gal_type, 'halo_id': halo_id,
                'halo_m' + mdef: self.mass[local], 'halo_r' + mdef: self.radius[local],
                'halo_num_centrals': counts[local], 'halo_num_satellites': counts[n + local],
                'host_centric_distance': hcd, 'conc_NFWmodel': self.conc[local]}
        for d, ax in enumerate('xyz'):
            data['halo_' + ax] = self.pos[local, d]
            data['halo_v' + ax] = self.vel[local, d]
        return data, ncen, ngal


class PopulatedHaloCatalog(ArrayCatalog):
    """
    The galaxies :meth:`HaloCatalog.populate` placed in a halo catalogue; :meth:`repopulate` draws them again in place.
    All columns are device tensors.
    """

    @CurrentMPIComm.enable
    def __init__(self, data, model, cosmo, comm=None):
        ArrayCatalog.__init__(self, data, comm=comm)
        self.model = model
        self.cosmo = cosmo

    @classmethod
    def _populate(cls, halos, model, seed, cosmo, comm, occ=None, into=None):
        data, ncen, ngal = halos.run(model, seed, occ)
        if into is None:
            into = cls.__new__(cls)
        else:
            into._overrides = {}
            into._attrs = {}
            for k in ('_csize',):
                into.__dict__.pop(k, None)
        PopulatedHaloCatalog.__init__(into, data, model, cosmo, comm=comm)
        into._halos = halos
        if into.csize == 0:
            raise ValueError("no particles in catalog after populating halo catalog")
        nsat = int(comm.allreduce(ngal - ncen))
        into.attrs.update(halos.attrs)
        into.attrs.update(model.param_dict)
        into.attrs.update(model.arguments())
        into.attrs['seed'] = seed
        into.attrs['gal_types'] = {t: i for i, t in enumerate(model.gal_types)}
        into.attrs['fsat'] = float(nsat) / into.csize
        return into

    def repopulate(self, seed=None, **params):
        """
        Draw the galaxies again, in place, with ``seed`` and updated model parameters.  The halo columns stay on the
        device from the first population; the same seed and parameters give the same catalogue, bit for bit.
        """
        model = _as_model(self.model)
        model.update(params)
        model.check()
        seed = _seed(self.comm, seed)
        occ = _occupation(model, self._halos.attrs['redshift'])
        PopulatedHaloCatalog._populate(self._halos, model, seed, self.cosmo, self.comm, occ, into=self)
