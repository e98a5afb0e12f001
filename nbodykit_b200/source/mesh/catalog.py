"""
CatalogMesh -- a catalogue viewed as a mesh (API of nbodykit/source/mesh/catalog.py), painted by the
CUDA scatter kernels, plus the window-compensation transfer functions (:419-594).

Differences from the reference's `to_real_field` (:155-403), none of which change results beyond
floating-point summation order:
  * no 4 Mi-particle chunk loop with per-chunk decompose / 3 Alltoallv / gc.collect(): the whole local
    catalogue (already in HBM, or copied there once) is routed and painted in one pass;
    `paint_chunk_size` is honoured only as the staging granularity for host-resident columns;
  * unit Weight/Value columns are never materialised (the kernel runs without a mass pointer);
  * interlacing paints both meshes in ONE pass over the particles;
  * `to_complex_field` (used by FFTPower through `compute(mode='complex')`) folds the 1+delta
    normalisation into the FFT scale and, when interlaced, skips the reference's c2r -> r2c round trip.
"""
import logging
import warnings

import numpy
import torch

from ... import _global_options, _lib
from ..._lib import check, lib, stage
from ...base.catalog import Column, ConstantColumn
from ...base.mesh import MeshSource
from ...pmesh import window
from ...pmesh.pm import ComplexField, RealField, _ptr, _stream, as_device_tensor, current_device


class CatalogMesh(MeshSource):
    """
    Parameters
    ----------
    source : CatalogSource
    Nmesh, BoxSize, dtype : mesh geometry / real dtype ('f4' | 'f8')
    Position, Weight, Value, Selection : columns (re-assignable attributes)
    interlaced : bool      Sefusatti et al. 2015 interlacing
    compensated : bool     divide out the window in Fourier space
    resampler : str        'cic', 'tsc', 'pcs', 'nnb'
    """
    logger = logging.getLogger('CatalogMesh')

    def __repr__(self):
        return "(%s as CatalogMesh)" % repr(self.source)

    def __init__(self, source, Nmesh, BoxSize, Position, dtype='f4', Weight=None, Value=None, Selection=None,
                 interlaced=False, compensated=False, resampler='cic', window=None):
        if window is not None:
            resampler = window
            warnings.warn("the window argument is deprecated; use resampler", DeprecationWarning)
        _Nmesh = numpy.empty(3, dtype='i8')
        _Nmesh[...] = Nmesh
        _BoxSize = numpy.empty(3, dtype='f8')
        _BoxSize[...] = BoxSize
        self.source = source
        self.Position = Position
        self.Selection = Selection
        self.Weight = Weight
        self.Value = Value
        self.attrs.update(source.attrs)
        self.attrs['interlaced'] = interlaced
        self.attrs['compensated'] = compensated
        self.attrs['resampler'] = str(resampler)
        MeshSource.__init__(self, source.comm, _Nmesh, _BoxSize, dtype)

    # ---- properties with setters (catalog.py:98-152)
    @property
    def interlaced(self):
        return self.attrs['interlaced']

    @interlaced.setter
    def interlaced(self, interlaced):
        self.attrs['interlaced'] = interlaced

    @property
    def window(self):
        warnings.warn("the window attribute is deprecated; use resampler", DeprecationWarning)
        return self.resampler

    @window.setter
    def window(self, value):
        self.resampler = value

    @property
    def resampler(self):
        return self.attrs['resampler']

    @resampler.setter
    def resampler(self, value):
        assert value in window.methods
        self.attrs['resampler'] = value

    @property
    def compensated(self):
        return self.attrs['compensated']

    @compensated.setter
    def compensated(self, value):
        self.attrs['compensated'] = value

    # ---- column staging
    def _device_columns(self):
        """Position (n,3) device tensor, mass (device tensor | scalar), plus N, W, W2 of the selection"""
        dev = current_device()

        def arr(col):
            if col is None:
                return None
            if isinstance(col, ConstantColumn):
                return col
            return col.compute() if isinstance(col, Column) else col

        pos = arr(self.Position)
        if isinstance(pos, ConstantColumn):
            pos = pos.materialize()
        sel, wgt, val = arr(self.Selection), arr(self.Weight), arr(self.Value)
        pos = as_device_tensor(pos, device=dev)
        if pos.dtype not in (torch.float32, torch.float64):
            pos = pos.to(torch.float64)
        mask = None
        if sel is not None:
            if isinstance(sel, ConstantColumn):
                if not bool(sel.value):
                    mask = torch.zeros(pos.shape[0], dtype=torch.bool, device=dev)
            else:
                mask = as_device_tensor(sel, device=dev).bool()
        if mask is not None:
            pos = pos[mask]
        n = int(pos.shape[0])

        def col_or_scalar(c):
            if c is None:
                return 1.0
            if isinstance(c, ConstantColumn):
                return float(c.value)
            t = as_device_tensor(c, device=dev)
            if t.dtype not in (torch.float32, torch.float64):
                t = t.to(torch.float64)
            return t[mask] if mask is not None else t

        w = col_or_scalar(wgt)
        v = col_or_scalar(val)
        # N, W = sum w, W2 = sum w^2 over WEIGHTS only (catalog.py:264-267)
        if isinstance(w, float):
            W, W2 = w * n, w * w * n
        else:
            acc = torch.zeros(2, dtype=torch.float64, device=dev)
            check(lib().nbk_sum_w_w2(_ptr(w), 4 if w.dtype == torch.float32 else 8, n, _ptr(acc), _stream()), "nbk_sum_w_w2")
            W, W2 = [float(x) for x in acc.cpu().tolist()]
        if isinstance(w, float) and isinstance(v, float):
            mass = w * v
        elif isinstance(w, float):
            mass = v if w == 1.0 else v * w
        elif isinstance(v, float):
            mass = w if v == 1.0 else w * v
        else:
            mass = w.to(torch.float64) * v.to(torch.float64) if w.dtype != v.dtype else w * v
        return pos, mass, n, W, W2

    def _host_streamed_paint(self):
        """Host-resident positions with unit weights on one GPU: copy in `paint_chunk_size`-sized pieces on a side
        stream and scatter each piece (usual tiled / direct dispatch, first piece clears the mesh) while the next one is in flight, so the paint hides behind
        the PCIe transfer instead of following it.  Returns None when the catalogue does not qualify."""
        pm = self.pm
        if pm.comm.size != 1:
            return None
        pos = self.Position.compute() if isinstance(self.Position, Column) and not isinstance(self.Position, ConstantColumn) else None
        if pos is None or (isinstance(pos, torch.Tensor) and pos.is_cuda):
            return None
        for c in (self.Weight, self.Value):
            if c is not None and not (isinstance(c, ConstantColumn)):
                return None
        if self.Selection is not None and not (isinstance(self.Selection, ConstantColumn) and bool(self.Selection.value)):
            return None
        t = pos if isinstance(pos, torch.Tensor) else torch.from_numpy(numpy.ascontiguousarray(pos))
        if t.dtype not in (torch.float32, torch.float64) or t.ndim != 2 or t.shape[1] != 3 or not t.is_contiguous():
            return None
        n = int(t.shape[0])
        chunk = 4 * int(_global_options['paint_chunk_size'])
        if n < 2 * chunk:
            return None
        resampler = window.methods[self.resampler]
        w = float(self.Weight.value) if self.Weight is not None else 1.0
        v = float(self.Value.value) if self.Value is not None else 1.0
        dev = current_device()
        main = torch.cuda.current_stream()
        side = torch.cuda.Stream(device=dev)
        reals = [RealField(pm)] + ([RealField(pm)] if self.interlaced else [])    # cleared by the first chunk's paint
        bufs = [torch.empty((chunk, 3), dtype=t.dtype, device=dev) for _ in range(2)]
        free = [torch.cuda.Event(), torch.cuda.Event()]
        for k, lo in enumerate(range(0, n, chunk)):
            hi = min(n, lo + chunk)
            b = bufs[k % 2]
            with torch.cuda.stream(side):
                side.wait_event(free[k % 2])                 # the scatter that last used this buffer is done
                b[:hi - lo].copy_(t[lo:hi], non_blocking=True)
                ready = torch.cuda.Event()
                ready.record(side)
            main.wait_event(ready)
            if self.interlaced:
                pm.paint_interlaced(b[:hi - lo], None, resampler, reals[0], reals[1], hold=(k > 0))
            else:
                pm.paint(b[:hi - lo], mass=1.0, resampler=resampler, hold=(k > 0), out=reals[0])
            free[k % 2].record(main)
        if w * v != 1.0:
            for r in reals:
                r *= (w * v)
        painted = tuple(reals) if self.interlaced else reals[0]
        return painted, n, w * n, w * w * n

    def _paint_raw(self):
        """un-normalised paint: returns (real | (real1, real2) if interlaced, N, W, W2)"""
        pm = self.pm
        resampler = window.methods[self.resampler]
        streamed = self._host_streamed_paint()
        if streamed is not None:
            return streamed
        with stage("H:columns"):
            pos, mass, Nlocal, Wlocal, W2local = self._device_columns()
        smoothing = (1.0 if self.interlaced else 0.5) * resampler.support
        scalar = isinstance(mass, float)
        # every rank paints its own particles (out-of-slab stencil points are dropped by the kernel) plus the
        # copies other ranks send for planes it owns
        batches = [(pos, mass)]
        if pm.comm.size > 1:
            with stage("H:decompose"):
                lay = pm.decompose(pos, smoothing=smoothing)
            with stage("H:route"):
                rpos, rmass = lay.route(pos, None if scalar else mass)
            batches.append((rpos, mass if scalar else rmass))
            with stage("H:allreduce3"):
                N, W, W2 = pm.comm.allreduce_floats([Nlocal, Wlocal, W2local])
            N = int(round(N))
        else:
            N, W, W2 = Nlocal, Wlocal, W2local
        if not self.interlaced:
            with stage("H:paint_all"):
                real = RealField(pm)
                first = True          # the first batch clears the mesh inside its own bucketing pass
                for p, m in batches:
                    if p.shape[0]:
                        pm.paint(p, mass=m, resampler=resampler, hold=not first, out=real)
                        first = False
                if first:
                    real[...] = 0
            return real, N, W, W2
        real1, real2 = RealField(pm), RealField(pm)
        first = True
        for p, m in batches:
            if p.shape[0]:
                pm.paint_interlaced(p, None if scalar else m, resampler, real1, real2, hold=not first)
                first = False
        if first:
            real1[...] = 0
            real2[...] = 0
        if scalar and mass != 1.0:
            real1 *= mass
            real2 *= mass
        return (real1, real2), N, W, W2

    def _attrs_for(self, N, W, W2):
        pm = self.pm
        nbar = 1. * W / numpy.prod(pm.Nmesh)
        if N == 0:
            warnings.warn(("trying to paint particle source to mesh, "
                           "but no particles were found!"), RuntimeWarning)
        with numpy.errstate(invalid='ignore', divide='ignore'):
            shotnoise = numpy.prod(pm.BoxSize) * W2 / W ** 2 if W != 0 else numpy.nan
        attrs = {}
        attrs['shotnoise'] = shotnoise
        attrs['N'] = N
        attrs['W'] = W
        attrs['W2'] = W2
        attrs['num_per_cell'] = nbar
        return attrs, nbar

    def to_real_field(self, out=None, normalize=True):
        """paint the density field; returns a RealField normalised to 1+delta (catalog.py:155-403);
        attrs: N, W, W2, shotnoise, num_per_cell"""
        pm = self.pm
        painted, N, W, W2 = self._paint_raw()
        if self.interlaced:
            real1, real2 = painted
            c1 = real1.r2c()
            c2 = real2.r2c()
            c1.interlace_combine(c2)
            del c2, real2
            c1.c2r(real1)
            painted = real1
        if out is not None:
            assert isinstance(out, RealField), "output of to_real_field must be a RealField"
            numpy.testing.assert_array_equal(out.pm.Nmesh, pm.Nmesh)
            toret = out
            toret += painted
        else:
            toret = painted
        attrs, nbar = self._attrs_for(N, W, W2)
        toret.attrs = attrs
        if pm.comm.rank == 0:
            self.logger.info("painted %d objects to mesh" % N)
            self.logger.info("mean particles per cell is %g", nbar)
        if normalize:
            if nbar > 0:
                toret /= nbar
            else:
                toret[...] = 1
            if pm.comm.rank == 0:
                self.logger.info("normalized the convention to 1 + delta")
        return toret

    def to_complex_field(self, out=None, x_pending=False):
        """FFT of the 1+delta field without the intermediate normalisation / interlacing round trip:
        complex = r2c(paint) / nbar (and the interlaced combination formed directly in Fourier space).
        x_pending=True (FFTPower's fused x pass and binning): where RealField._r2c_zy applies to a non-interlaced
        mesh, the field is returned after the z and y passes only, with `_x_scale` = 1/nbar, the factor the x pass
        still owes on top of 1/prod(Nmesh); a complete field has no `_x_scale`."""
        painted, N, W, W2 = self._paint_raw()
        attrs, nbar = self._attrs_for(N, W, W2)
        c = painted._r2c_zy() if (x_pending and nbar > 0 and not self.interlaced) else None
        if c is not None:
            c._x_scale = 1.0 / nbar
        elif nbar <= 0:
            real = painted[0] if self.interlaced else painted
            real[...] = 1
            c = real.r2c()
        elif self.interlaced:
            real1, real2 = painted
            c = real1.r2c(scale=1.0 / nbar)          # normalisation folded into the FFT's last pass
            c2 = real2.r2c(scale=1.0 / nbar)
            c.interlace_combine(c2)
        else:
            with stage("H:r2c"):
                c = painted.r2c(scale=1.0 / nbar)
        c.attrs = attrs
        if self.pm.comm.rank == 0:
            self.logger.info("painted %d objects to mesh" % N)
        return c

    def compute_complex_deferred(self, Nmesh=None, x_pending=False):
        """FFTPower fast path: (complex field WITHOUT the window compensation, name of the compensation the
        caller must still apply) when the compensation is the only action -- the power-binning kernel then
        applies it on the fly.  Falls back to (compute('complex', Nmesh=Nmesh), None) -- also whenever another
        mesh size is asked for (the resampling of MeshSource.compute applies).  x_pending: see to_complex_field."""
        own = self._get_compensation() if self.compensated else []
        other_n = Nmesh is not None and any(numpy.ones(3, dtype='i8') * Nmesh != self.attrs['Nmesh'])
        if list(MeshSource.actions.fget(self)) or not own or other_n:
            return self.compute(mode='complex', Nmesh=Nmesh), None
        c = self.to_complex_field(x_pending=x_pending)
        c.attrs.update(self.attrs)
        return c, own[0][1].__name__

    @property
    def actions(self):
        """actions applied to the density field, with the compensation first (catalog.py:405-417)"""
        actions = MeshSource.actions.fget(self)
        if self.compensated:
            actions = self._get_compensation() + actions
        return actions

    def _get_compensation(self):
        return get_compensation(self.interlaced, self.resampler)


def get_compensation(interlaced, resampler):
    """the compensation action for a window: sinc^p de-convolution when interlaced, the
    shot-noise-aware form of Jing et al. 2005 otherwise (catalog.py:419-447)"""
    if interlaced:
        d = {'cic': CompensateCIC, 'tsc': CompensateTSC, 'pcs': CompensatePCS}
    else:
        d = {'cic': CompensateCICShotnoise, 'tsc': CompensateTSCShotnoise, 'pcs': CompensatePCSShotnoise}
    if resampler not in d:
        raise ValueError("compensation for window %s is not defined" % resampler)
    return [('complex', d[resampler], "circular")]


# ---------------------------------------------------------------------------------------------------
# Transfer functions f(w, v): `w` = three broadcastable circular-frequency arrays in [-pi, pi), `v` the
# field values.  When applied through MeshSource / Field.apply they run as the CUDA kernel
# nbk_compensate (same name -> same formula); the NumPy bodies below serve direct calls on host arrays.
# ---------------------------------------------------------------------------------------------------
def _sinc_compensation(w, v, p):
    for i in range(3):
        wi = w[i]
        tmp = (numpy.sinc(0.5 * wi / numpy.pi)) ** p
        tmp[wi == 0.] = 1.
        v = v / tmp
    return v


def CompensateTSC(w, v):
    """divide by sinc^3 per axis: TSC window (Jing et al 2005), for interlaced fields"""
    return _sinc_compensation(w, v, 3)


def CompensatePCS(w, v):
    """divide by sinc^4 per axis: PCS window, for interlaced fields"""
    return _sinc_compensation(w, v, 4)


def CompensateCIC(w, v):
    """divide by sinc^2 per axis: CIC window, for interlaced fields"""
    return _sinc_compensation(w, v, 2)


def CompensateTSCShotnoise(w, v):
    """TSC window with the first-order aliasing (shot-noise) correction of Jing et al 2005"""
    for i in range(3):
        s = numpy.sin(0.5 * w[i]) ** 2
        v = v / (1 - s + 2. / 15 * s ** 2) ** 0.5
    return v


def CompensatePCSShotnoise(w, v):
    """PCS window with the aliasing correction (polynomial fitted in s = sin^2(w/2))"""
    for i in range(3):
        s = numpy.sin(0.5 * w[i]) ** 2
        v = v / (1 - 4. / 3. * s + 2. / 5. * s ** 2 - 4. / 315. * s ** 3) ** 0.5
    return v


def CompensateCICShotnoise(w, v):
    """CIC window with the aliasing correction of Jing et al 2005"""
    for i in range(3):
        v = v / (1 - 2. / 3 * numpy.sin(0.5 * w[i]) ** 2) ** 0.5
    return v
