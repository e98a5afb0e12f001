"""
FFTPower -- periodic-box P(k), P(k,mu), P_ell(k)   (mirrors nbodykit/algorithms/fftpower.py).

Same constructor, attrs, `.power` / `.poles` BinnedStatistic results, `.run()`, `.save()`, `.load()`
as the reference (fftpower.py:146-359).  What differs is where the O(Nmesh^3) work runs:

  reference                                   here
  ------------------------------------------  ------------------------------------------------------
  _compute_3d_power: 3 python slab passes     fused into the binning kernel (no p3d field is written)
  (c1*conj(c2), zero mode, *V)  :91-143
  project_to_basis: ~15 NumPy passes per      nbk_power_bin: one read of c1 (and c2), float32 coordinate
  x-slab + 4 MPI allreduce      :507-701      arithmetic bit-identical to the reference's digitize, f64
                                              accumulators, one NCCL all-reduce of the packed histogram
"""
import logging

import numpy
import torch

from .. import CurrentMPIComm, _lib
from .._lib import check, lib, stage
from ..binned_statistic import BinnedStatistic
from ..base.catalog import CatalogSourceBase
from ..base.mesh import MeshSource
from ..pmesh.pm import ComplexField, Field, RealField, _ptr, _stream, _CODE


class FFTBase(object):
    """base of the periodic FFT power spectrum algorithms (fftpower.py:12-143)"""

    def __init__(self, first, second, Nmesh, BoxSize):
        first = _cast_source(first, Nmesh=Nmesh, BoxSize=BoxSize)
        if second is not None:
            second = _cast_source(second, Nmesh=Nmesh, BoxSize=BoxSize)
        else:
            second = first
        self.first = first
        self.second = second
        self.comm = first.comm
        assert second.comm is first.comm, "communicator mismatch between input sources"
        if not numpy.array_equal(first.attrs['BoxSize'], second.attrs['BoxSize']):
            raise ValueError("'BoxSize' mismatch between sources in FFTPower")
        self.attrs = {}
        self.attrs['Nmesh'] = first.attrs['Nmesh'].copy()
        self.attrs['BoxSize'] = first.attrs['BoxSize'].copy()
        self.attrs.update(zip(['Lx', 'Ly', 'Lz'], self.attrs['BoxSize']))
        self.attrs.update({'volume': self.attrs['BoxSize'].prod()})

    def save(self, output):
        """save the result as JSON (same state layout as the reference, fftpower.py:57-69)"""
        import json
        from ..utils import JSONEncoder
        if self.comm.rank == 0:
            self.logger.info('measurement done; saving result to %s' % output)
            with open(output, 'w') as ff:
                json.dump(self.__getstate__(), ff, cls=JSONEncoder)

    @classmethod
    @CurrentMPIComm.enable
    def load(cls, output, comm=None):
        import json
        from ..utils import JSONDecoder
        if comm.rank == 0:
            with open(output, 'r') as ff:
                state = json.load(ff, cls=JSONDecoder)
        else:
            state = None
        state = comm.bcast(state)
        self = object.__new__(cls)
        self.__setstate__(state)
        self.comm = comm
        return self

    def _compute_3d_power(self, first, second):
        """the two complex fields whose product is the 3-D power, plus attrs (fftpower.py:91-143).
        The product c1*conj(c2)*V with the zero mode cleared is formed inside the binning kernel."""
        attrs = {}
        attrs.update(self.attrs)

        def field_of(src):
            # a CatalogMesh whose only action is its window compensation hands over the uncompensated field
            # and the name of the transfer function; the binning kernel applies it on the fly
            if hasattr(src, 'compute_complex_deferred'):
                return src.compute_complex_deferred(Nmesh=self.attrs['Nmesh'])
            return src.compute(mode='complex', Nmesh=self.attrs['Nmesh']), None
        c1, comp1 = field_of(first)
        if first is second:
            c2, comp2 = c1, comp1
        else:
            c2, comp2 = field_of(second)
        self._deferred_compensation = (comp1, comp2)
        N1 = c1.attrs.get('N', 0)
        N2 = c2.attrs.get('N', 0)
        attrs.update({'N1': N1, 'N2': N2})
        Pshot = 0
        if self.first is self.second:
            if 'shotnoise' in c1.attrs:
                Pshot = c1.attrs['shotnoise']
        attrs['shotnoise'] = Pshot
        return c1, c2, attrs


class FFTPower(FFTBase):
    """
    Power spectrum of one or two sources in a periodic box: 1-D P(k) or 2-D P(k,mu), plus
    multipoles (fftpower.py:146-359).  Results are computed in __init__ and stored as
    `.power`, `.poles` (BinnedStatistic) and `.attrs`.  Shot noise is NOT subtracted.
    """
    logger = logging.getLogger('FFTPower')

    def __init__(self, first, mode, Nmesh=None, BoxSize=None, second=None,
                 los=[0, 0, 1], Nmu=5, dk=None, kmin=0., kmax=None, poles=[]):
        if mode not in ['1d', '2d']:
            raise ValueError("`mode` should be either '1d' or '2d'")
        if poles is None:
            poles = []
        if numpy.isscalar(los) or len(los) != 3:
            raise ValueError("line-of-sight ``los`` should be vector with length 3")
        if not numpy.allclose(numpy.einsum('i,i', los, los), 1.0, rtol=1e-5):
            raise ValueError("line-of-sight ``los`` must be a unit vector")
        FFTBase.__init__(self, first, second, Nmesh, BoxSize)
        self.attrs['mode'] = mode
        self.attrs['los'] = los
        self.attrs['Nmu'] = Nmu
        self.attrs['poles'] = poles
        if dk is None:
            dk = 2 * numpy.pi / self.attrs['BoxSize'].min()
        self.attrs['dk'] = dk
        self.attrs['kmin'] = kmin
        self.attrs['kmax'] = kmax
        self.power, self.poles = self.run()
        self.attrs.update(self.power.attrs)

    def run(self):
        if self.attrs['mode'] == "1d":
            self.attrs['Nmu'] = 1
        with stage("H:compute_fields"):
            c1, c2, attrs = self._compute_3d_power(self.first, self.second)
        dk = self.attrs['dk']
        kmin = self.attrs['kmin']
        kmax = self.attrs['kmax']
        if kmax is None:
            kmax = numpy.pi * c1.Nmesh.min() / c1.BoxSize.max() + dk / 2
        if dk > 0:
            kedges = numpy.arange(kmin, kmax, dk)
            kcoords = None
        else:
            kedges, kcoords = _find_unique_edges(c1.pm, kmax)
        muedges = numpy.linspace(-1, 1, self.attrs['Nmu'] + 1, endpoint=True)
        edges = [kedges, muedges]
        coords = [kcoords, None]
        result, pole_result = project_to_basis_device(
            c1, edges, poles=self.attrs['poles'], los=self.attrs['los'], second=None if c2 is c1 else c2,
            is_p3d=False, volume=float(self.attrs['BoxSize'].prod()), compensation=self._deferred_compensation,
            need_mu=(self.attrs['mode'] != "1d"))

        if self.attrs['mode'] == "1d":
            cols = ['k', 'power', 'modes']
            icols = [0, 2, 3]
            edges = edges[0:1]
            coords = coords[0:1]
        else:
            cols = ['k', 'mu', 'power', 'modes']
            icols = [0, 1, 2, 3]
        dtype = numpy.dtype([(name, result[icol].dtype.str) for icol, name in zip(icols, cols)])
        power = numpy.squeeze(numpy.empty(result[0].shape, dtype=dtype))
        for icol, col in zip(icols, cols):
            power[col][:] = numpy.squeeze(result[icol])

        poles = None
        if pole_result is not None:
            k, poles, N = pole_result
            cols = ['k'] + ['power_%d' % l for l in self.attrs['poles']] + ['modes']
            result = [k] + [pole for pole in poles] + [N]
            dtype = numpy.dtype([(name, result[icol].dtype.str) for icol, name in enumerate(cols)])
            poles = numpy.empty(result[0].shape, dtype=dtype)
            for icol, col in enumerate(cols):
                poles[col][:] = result[icol]
        return self._make_datasets(edges, poles, power, coords, attrs)

    def __getstate__(self):
        return dict(power=self.power.__getstate__(),
                    poles=self.poles.__getstate__() if self.poles is not None else None,
                    attrs=self.attrs)

    def __setstate__(self, state):
        self.attrs = state['attrs']
        self.power = BinnedStatistic.from_state(state['power'])
        self.poles = None
        if state['poles'] is not None:
            self.poles = BinnedStatistic.from_state(state['poles'])

    def _make_datasets(self, edges, poles, power, coords, attrs):
        if self.attrs['mode'] == '1d':
            power = BinnedStatistic(['k'], edges, power, fields_to_sum=['modes'], coords=coords, **attrs)
        else:
            power = BinnedStatistic(['k', 'mu'], edges, power, fields_to_sum=['modes'], coords=coords, **attrs)
        if poles is not None:
            poles = BinnedStatistic(['k'], [power.edges['k']], poles, fields_to_sum=['modes'],
                                    coords=[power.coords['k']], **attrs)
        return power, poles


class ProjectedFFTPower(FFTBase):
    """
    Power spectrum of a field projected (summed) over one or two axes of the box -- the "1d" / "2d" power of
    Lyman-alpha forest or lensing maps (fftpower.py:361-505).  The 3-D work (paint, r2c, Fourier-space actions, c2r
    and the projection) runs on the device; what is left is a 1-D / 2-D FFT of Nmesh or Nmesh^2 numbers, done on
    the host with numpy exactly as the reference does.  Results: `.edges`, `.power` (BinnedStatistic with k, power,
    modes), computed in __init__.
    """
    logger = logging.getLogger('ProjectedFFTPower')

    def __init__(self, first, Nmesh=None, BoxSize=None, second=None, axes=(0, 1), dk=None, kmin=0.):
        FFTBase.__init__(self, first, second, Nmesh, BoxSize)
        assert len(axes) in (1, 2), "length of ``axes`` in ProjectedFFTPower should be 1 or 2"
        if dk is None:
            dk = 2 * numpy.pi / self.attrs['BoxSize'].min()
        self.attrs['dk'] = dk
        self.attrs['kmin'] = kmin
        self.attrs['axes'] = axes
        self.run()

    def _projected_modes(self, source):
        """rfftn of the real field summed over the axes that are not kept, normalised by prod(Nmesh)"""
        c = source.compute(Nmesh=self.attrs['Nmesh'], mode='complex')
        r = c.c2r().preview(axes=self.attrs['axes'])
        return numpy.fft.rfftn(r) / self.attrs['Nmesh'].prod()

    def run(self):
        c1 = self._projected_modes(self.first)
        c2 = c1 if self.first is self.second else self._projected_modes(self.second)
        pk = c1 * c2.conj()
        pk.flat[0] = 0
        axes = list(self.attrs['axes'])
        shape = numpy.array([self.attrs['Nmesh'][i] for i in axes], dtype='int')
        boxsize = numpy.array([self.attrs['BoxSize'][i] for i in axes])
        # broadcastable wavenumbers of the kept axes (the last one is Hermitian-compressed)
        k = []
        for d, (N, L) in enumerate(zip(shape, boxsize)):
            kd = numpy.fft.fftfreq(N, 1. / (N * 2 * numpy.pi / L))[:pk.shape[d]]
            sh = [1] * len(shape)
            sh[d] = -1
            k.append(kd.reshape(sh))
        kmag = sum(ki ** 2 for ki in k) ** 0.5
        # Hermitian weights along the compressed axis: 2, except its first and last plane
        W = numpy.empty(pk.shape, dtype='f4')
        W[...] = 2.0
        W[..., 0] = 1.0
        W[..., -1] = 1.0
        dk, kmin = self.attrs['dk'], self.attrs['kmin']
        kedges = numpy.arange(kmin, numpy.pi * self.attrs['Nmesh'][axes].min() / self.attrs['BoxSize'][axes].max() + dk / 2, dk)
        nb = len(kedges) + 1
        dig = numpy.digitize(kmag.flat, kedges)
        xsum = numpy.bincount(dig, weights=(W * kmag).flat, minlength=nb).astype('f8')
        Psum = numpy.bincount(dig, weights=(W * pk.real).flat, minlength=nb) \
            + 1j * numpy.bincount(dig, weights=(W * pk.imag).flat, minlength=nb)
        Nsum = numpy.bincount(dig, weights=W.flat, minlength=nb).astype('f8')
        power = numpy.empty(len(kedges) - 1, dtype=[('k', 'f8'), ('power', 'c16'), ('modes', 'f8')])
        with numpy.errstate(invalid='ignore', divide='ignore'):
            power['k'] = (xsum / Nsum)[1:-1]
            power['power'] = (Psum / Nsum)[1:-1] * boxsize.prod()     # dimension is 'volume' of the kept axes
            power['modes'] = Nsum[1:-1]
        self.edges = kedges
        self.power = BinnedStatistic(['k'], [self.edges], power)

    def __getstate__(self):
        return dict(edges=self.edges, power=self.power.data, attrs=self.attrs)

    def __setstate__(self, state):
        self.__dict__.update(state)
        self.power = BinnedStatistic(['k'], [self.edges], self.power)


def _los_coord_mode(los, coord_dtype):
    """which arithmetic `MeshSlab.mu` runs in (meshtools.py:136): with float32 coordinate arrays,
    Python-number los components keep mu in float32, NumPy float64 components promote it to float64
    (NumPy >= 2 promotion rules)."""
    if coord_dtype in ("f8", 8):
        return 8
    strong = any(isinstance(v, (numpy.floating, numpy.ndarray)) and numpy.asarray(v).dtype == numpy.float64
                 for v in los)
    return 48 if strong else 4


def project_to_basis_device(y3d, edges, los=[0, 0, 1], poles=[], coord_dtype="f4", is_p3d=True, second=None,
                            volume=1.0, compensation=(None, None), clear_zero=True, antihermitian=False, mirror=None,
                            need_mu=True):
    """
    project_to_basis (fftpower.py:507-701) for a device ComplexField.

    With ``is_p3d=True`` `y3d` is the 3-D statistic itself (reference semantics).  With
    ``is_p3d=False`` the statistic is `y3d * conj(second or y3d) * volume` with the k=0 mode
    cleared, formed on the fly (fftpower.py:115-128) -- the FFTPower fast path; `compensation` then names
    the window transfer functions (`Compensate*`) still to be divided out of `y3d` / `second`, also on the fly.
    ``antihermitian=True``: the statistic obeys y(-k) = -conj y(k) (odd FKP multipoles A0 conj(A_l)); the mirror half
    of the compressed field is folded in with that sign, which is what a full complex ('c16') mesh gives the reference.

    Returns exactly what the reference returns:
    ``(xmean_2d, mumean_2d, y2d, N_2d), (xmean_1d, poles, N_1d) | None``.
    """
    is_real = isinstance(y3d, RealField)
    if not isinstance(y3d, (ComplexField, RealField)):
        raise TypeError("project_to_basis_device needs a RealField or ComplexField")
    if is_real and not is_p3d:
        raise ValueError("a RealField is binned as a 3-D statistic (is_p3d=True)")
    pm = y3d.pm
    if second is not None and second is not y3d:
        # the kernel reads both fields with ONE dtype code and ONE slab geometry: anything else must not reach it
        if not isinstance(second, type(y3d)):
            raise TypeError("project_to_basis_device: the two fields must be of the same kind (real / complex)")
        if not numpy.array_equal(second.pm.Nmesh, pm.Nmesh) or tuple(second.value.shape) != tuple(y3d.value.shape):
            raise ValueError("project_to_basis_device: mesh shape mismatch between the two fields (%s vs %s)"
                             % (str(tuple(second.value.shape)), str(tuple(y3d.value.shape))))
        if second.pm.typestr != pm.typestr:
            # the reference multiplies c1 * conj(c2) under NumPy promotion: promote the narrower field (a copy)
            if pm.typestr == 'f8':
                second = type(second)(pm, second.value.to(y3d.value.dtype))
            else:
                y3d = type(y3d)(second.pm, y3d.value.to(second.value.dtype))
                pm = y3d.pm
    # real-space statistics (FFTCorr) are binned in the wrapped separation x = index * L/N
    coord_unit = _lib.darr(pm.BoxSize / pm.Nmesh) if is_real else None
    comm = pm.comm
    xedges, muedges = edges
    # edges**2 is formed in the dtype the edges come in (fftpower.py:583 `x2edges = xedges**2`: float32 for the
    # dk = 0 edges, which are built from float32 coordinates) and only then widened -- the widening is exact
    x2edges = (numpy.asarray(xedges) ** 2).astype('f8')
    xedges = numpy.asarray(xedges, dtype='f8')
    muedges = numpy.asarray(muedges, dtype='f8')
    Nx = len(xedges) - 1
    Nmu = len(muedges) - 1
    poles = list(poles)
    do_poles = len(poles) > 0
    _poles = [0] + sorted(poles) if 0 not in poles else sorted(poles)
    if any(ell < 0 for ell in _poles):
        raise ValueError("in `project_to_basis`, multipole numbers must be non-negative integers")
    ell_idx = [_poles.index(l) for l in poles]
    Nell = len(_poles)
    nb = (Nx + 2) * (Nmu + 2)

    dev = y3d.value.device
    # one launch bins at most 8 multipoles (NBK_MAX_ELL), the first of them l = 0: any number of poles is binned in
    # groups, _poles[:8] and then [0] + the next 7, each group into its own rows of ysum.  The l = 0 row of every
    # further group repeats the first group's and is dropped.
    groups = [_poles[:8]] + [[0] + _poles[i:i + 7] for i in range(8, Nell, 7)]
    nrow = sum(len(grp) for grp in groups)
    # one packed accumulator: [xsum | musum | ysum(nrow*nb*2)] (and nsum) so a single all-reduce suffices
    nsum = torch.zeros(nb, dtype=torch.int64, device=dev)
    facc = torch.zeros(nb * (2 + 2 * nrow), dtype=torch.float64, device=dev)
    xsum = facc[:nb]
    musum = facc[nb:2 * nb]
    # the counts and k sums of the further groups repeat the first group's: they go to a scratch pair that is not reduced
    if len(groups) > 1:
        spare_n = torch.zeros(nb, dtype=torch.int64, device=dev)
        spare_x = torch.zeros(nb, dtype=torch.float64, device=dev)
    tr, start, count = (0, pm.x_start, pm.x_n) if is_real else y3d._slab()
    los_f = [float(v) for v in los]
    herm = 0 if (is_real or not y3d.compressed) else (2 if antihermitian else 1)
    if mirror is not None and (herm != 1 or second is None or tuple(mirror.value.shape) != tuple(y3d.value.shape)):
        raise ValueError("a mirror field needs a Hermitian-compressed pair of fields of the same shape")
    with stage("power_bin"):
        fn = lib().nbk_power_bin if mirror is None else lib().nbk_power_bin2
        extra = () if mirror is None else (_ptr(mirror.value),)
        row, keep = 0, []
        for i, grp in enumerate(groups):
            first = i == 0
            check(fn(
                _ptr(y3d.value), _ptr(second.value) if second is not None else None, *extra, _CODE[pm.typestr],
                1 if is_p3d else 0, float(volume), 1 if clear_zero else 0, pm._nmesh_c, pm._box_c, tr, start, count,
                _los_coord_mode(los, coord_dtype), _lib.darr(x2edges), Nx, _lib.darr(muedges), Nmu, _lib.darr(los_f),
                _lib.i32arr(grp), len(grp), herm, _lib.COMP.get(compensation[0], 0),
                _lib.COMP.get(compensation[1], 0), 1 if is_real else 0, coord_unit,
                _ptr(nsum if first else spare_n), _ptr(xsum if first else spare_x),
                _ptr(musum) if (need_mu and first) else None, _ptr(facc[(2 + 2 * row) * nb:]), _stream()),
                "nbk_power_bin")
            keep += range(row if first else row + 1, row + len(grp))
            row += len(grp)
    with stage("H:bin_reduce"):
        if comm.size > 1:
            comm.allreduce_tensor(nsum)
            comm.allreduce_tensor(facc)
        Nsum = nsum.cpu().numpy().reshape(Nx + 2, Nmu + 2)
        f = facc.cpu().numpy()
    xsum = f[:nb].reshape(Nx + 2, Nmu + 2)
    musum = f[nb:2 * nb].reshape(Nx + 2, Nmu + 2)
    ysum = f[2 * nb:].reshape(nrow, Nx + 2, Nmu + 2, 2)[keep]
    ysum = ysum[..., 0] + 1j * ysum[..., 1]

    # fold the mu == 1 overflow bin, form the means (fftpower.py:674-701)
    ysum[..., -2] += ysum[..., -1]
    musum[:, -2] += musum[:, -1]
    xsum[:, -2] += xsum[:, -1]
    Nsum[:, -2] += Nsum[:, -1]
    sl = slice(1, -1)
    with numpy.errstate(invalid='ignore', divide='ignore'):
        y2d = (ysum[0, ...] / Nsum)[sl, sl]
        xmean_2d = (xsum / Nsum)[sl, sl]
        mumean_2d = (musum / Nsum)[sl, sl]
        N_2d = Nsum[sl, sl]
        if do_poles:
            N_1d = Nsum[sl, sl].sum(axis=-1)
            xmean_1d = xsum[sl, sl].sum(axis=-1) / N_1d
            poles_ = ysum[:, sl, sl].sum(axis=-1) / N_1d
            poles_ = poles_[ell_idx, ...]
    result = (xmean_2d, mumean_2d, y2d, N_2d)
    pole_result = (xmean_1d, poles_, N_1d) if do_poles else None
    return result, pole_result


def project_to_basis(y3d, edges, los=[0, 0, 1], poles=[]):
    """reference-compatible entry point (fftpower.py:507): `y3d` is a 3-D statistic held in a ComplexField"""
    return project_to_basis_device(y3d, edges, los=los, poles=poles, is_p3d=True)


def _cast_source(source, BoxSize, Nmesh):
    """cast an object to a MeshSource (fftpower.py:703-730)"""
    from ..source.mesh import FieldMesh
    if isinstance(source, Field):
        source = FieldMesh(source)
    elif isinstance(source, CatalogSourceBase):
        if not isinstance(source, MeshSource):
            source = source.to_mesh(BoxSize=BoxSize, Nmesh=Nmesh, dtype='f8', compensated=True)
    if not isinstance(source, MeshSource):
        raise TypeError("Unknown type of source in FFTPower: %s" % str(type(source)))
    if BoxSize is not None and any(source.attrs['BoxSize'] != BoxSize):
        raise ValueError("Mismatched Boxsize between __init__ and source.attrs")
    if Nmesh is not None and any(source.attrs['Nmesh'] != Nmesh):
        raise ValueError(("Mismatched Nmesh between __init__ and source.attrs; "
                          "if trying to re-sample with a different mesh, specify "
                          "`Nmesh` as keyword of to_mesh()"))
    return source


def _find_unique_edges(pm, xmax, real=False):
    """`dk=0` / `dr=0`: one bin per distinct |k| (or, real=True, per distinct separation |x|) on the lattice
    (fftpower.py:732-769; fftcorr.py:167).

    The reference broadcasts a full x^2 array per rank and uniquifies it; the distinct values are the
    distinct sums of three squared 1-D coordinates, found here from the 1-D arrays alone (host, O(N^2)).
    Same quantisation: ix2 = int64(fx2 / (0.05 x0)^2 + 0.5), first occurrence kept."""
    N = [int(v) for v in pm.Nmesh]
    x0 = (pm.BoxSize / pm.Nmesh) if real else (2 * numpy.pi / pm.BoxSize)
    ct = numpy.float32                         # coordinate arrays of the fields are float32 (SURVEY B.5)
    full = []
    for d in range(3):
        n = N[d] if (real or d != 2) else pm.Nzc
        j = numpy.arange(n)
        j[j >= (N[d] + 1) // 2] -= N[d]
        full.append(j.astype(ct) * ct(x0[d]))
    binning = (x0.min() * 0.05) ** 2
    # Device pass over the planes in the reference's ravel order (x, y, z), keeping the first occurrence of every
    # quantised value: per plane a sort of ~N^2/2 keys, merged into the running set by a stable sort (earlier planes
    # first).  Planes whose x coordinate squares to a value already seen add nothing and are skipped.  The set has
    # ~3 (N/2)^2 members at most, so the whole pass takes well under a second at 1024^3.
    # (coordinate bookkeeping, not field data: it runs wherever torch runs, so the host-logic tests can pin it)
    dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
    fx_t = [torch.from_numpy(numpy.ascontiguousarray(f)).to(dev) for f in full]
    best_k = torch.empty(0, dtype=torch.int64, device=dev)
    best_v = torch.empty(0, dtype=torch.float32, device=dev)
    seen = set()
    for ix in range(len(full[0])):
        x2 = float(full[0][ix] * full[0][ix])
        if x2 in seen:
            continue
        seen.add(x2)
        # (0 + x^2 + y^2) + z^2 in float32, as the reference's sum(xi ** 2) associates it
        fx2 = ((0 + fx_t[0][ix] ** 2) + fx_t[1][:, None] ** 2 + fx_t[2][None, :] ** 2).reshape(-1)
        key = (fx2.double() / binning + 0.5).to(torch.int64)
        allk = torch.cat([best_k, key])
        allv = torch.cat([best_v, fx2])
        order = torch.sort(allk, stable=True).indices
        sk = allk[order]
        first = torch.ones_like(sk, dtype=torch.bool)
        first[1:] = sk[1:] != sk[:-1]
        best_k = sk[first]
        best_v = allv[order][first]
    fx = best_v.cpu().numpy() ** 0.5
    fx = fx[fx < xmax]
    # second pass of the reference (re-bin after allgather with bin size minx0*1e-5)
    ix = numpy.int64(fx / (x0.min() * 1e-5) + 0.5)
    _, ind = numpy.unique(ix, return_index=True)
    fx = fx[ind]
    width = numpy.diff(fx)
    edges = fx.copy()
    edges[1:] -= width * 0.5
    edges = numpy.append(edges, [fx[-1] + width[-1] * 0.5])
    edges[0] = 0
    return edges, fx
