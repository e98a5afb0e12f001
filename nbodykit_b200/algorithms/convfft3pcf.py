"""
ConvolvedFFT3PCF -- edge-corrected multipoles of the isotropic three-point correlation function of a survey catalogue on
the mesh, with FFTs (Slepian & Eisenstein, MNRAS 454, 4142 (2015) §4; MNRAS 455, L31 (2016); DESIGN.md 4.17).  The
survey counterpart of FFT3PCF, with ConvolvedFFTPower's FKP field and alpha.  The reference has no mesh 3PCF.

D and R are the data and randoms species fields painted as FKPCatalogMesh.to_real_field paints them (mass u = w_c w_fkp
Value, no compensation) and restricted to the window box (window_box: zero outside it, a no-op unless the mesh is
interlaced), N = (D - alpha R) / V_cell (no mean is subtracted: the padding stays zero) and Rf = alpha R / V_cell.
With true (non-periodic) grid separations and FFT3PCF's bins,

    nnn_l(b1, b2) = (2l + 1) / (16 pi^2) sum_x N(x) sum_{s1 in b1} sum_{s2 in b2} N(x + s1) N(x + s2) L_l(u1.u2)

and rrr_l the same with Rf; zeta = threeptcf.edge_correct(nnn, rrr, poles).  The geometry guard proves that no pair
within r_max wraps around the periodic mesh, so the periodic FFT sums are the true ones.  The bin loop is
fft3pcf.bin_pass with the two sources (N, N^) and (Rf, R^) sharing every kernel spectrum, and with the tile-listed Gram
(nbk_fft3pcf_gram_tiles) over the tiles where the weight field is nonzero.
"""
import logging

import numpy
import torch

from .. import CurrentMPIComm
from .._lib import stage
from ..binned_statistic import BinnedStatistic
from ..pmesh.window import FindResampler
from ..utils import JSONDecoder, JSONEncoder, get_data_bounds
from .convpower.fkp import _cast_mesh
from .fft3pcf import GRAM_TILE, bin_pass, separation_counts, tile_list
from .threeptcf import _check_edges, _check_poles, edge_correct


def check_contiguous_poles(poles):
    """the validated poles (threeptcf._check_poles), which must also be every ell from 0 to max(poles)"""
    p = _check_poles(poles)
    if sorted(p) != list(range(max(p) + 1)):
        raise ValueError("ConvolvedFFT3PCF: poles must hold every ell from 0 to max(poles) (got %s): the edge "
                         "correction couples all of them" % p)
    return p


def min_box_size(lo, hi, Nmesh, support, rmax):
    """per axis, the BoxSize the geometry guard needs: (hi - lo) + (support + 2) L / N + rmax < L and rmax <= L / 2.
    Returns the infimum of the passing L (inf where the mesh is too coarse for any L)."""
    N = numpy.asarray(Nmesh, dtype='f8')
    ext = numpy.asarray(hi, dtype='f8') - numpy.asarray(lo, dtype='f8')
    frac = 1.0 - (support + 2) / N
    with numpy.errstate(divide='ignore'):
        need = numpy.where(frac > 0, (ext + rmax) / numpy.where(frac > 0, frac, 1.0), numpy.inf)
    return numpy.maximum(need, 2 * rmax)


def geometry_guard(lo, hi, Nmesh, BoxSize, support, rmax):
    """raises ValueError unless, per axis i, (hi_i - lo_i) + (support + 2) H_i + rmax < L_i and rmax <= L_i / 2: then
    no pair of painted cells within rmax is joined through the periodic boundary.  support + 2 covers the window's
    stencil, its edge and the interlaced half-cell shift."""
    L = numpy.asarray(BoxSize, dtype='f8')
    H = L / numpy.asarray(Nmesh, dtype='f8')
    ext = numpy.asarray(hi, dtype='f8') - numpy.asarray(lo, dtype='f8')
    if ((ext + (support + 2) * H + rmax < L) & (rmax <= 0.5 * L)).all():
        return
    need = min_box_size(lo, hi, Nmesh, support, rmax)
    raise ValueError("ConvolvedFFT3PCF: the survey (extent %s) with max(edges) = %g does not fit the periodic mesh of "
                     "BoxSize %s without pairs wrapping; it needs BoxSize > %s at this Nmesh"
                     % (_fmt(ext), rmax, _fmt(L), _fmt(need)))


def window_box(lo, hi, H, support):
    """per axis the interval [a, b], relative to BoxCenter, that holds every cell node a window of `support` cells
    paints for positions in [lo, hi]: [lo - (support / 2 + 1) H, hi + (support / 2 + 1) H].  Its width is the
    (hi - lo) + (support + 2) H of the geometry guard."""
    m = (0.5 * support + 1) * numpy.asarray(H, dtype='f8')
    return numpy.asarray(lo, dtype='f8') - m, numpy.asarray(hi, dtype='f8') + m


def box_mask(Nmesh, BoxSize, a, b):
    """per axis a float64 vector over the cell index i: 1 where the node i H, wrapped into the box (positions are
    relative to BoxCenter and wrap with period L), lies in [a, b], else 0"""
    out = []
    for N, L, lo, hi in zip(numpy.broadcast_to(Nmesh, 3), numpy.broadcast_to(BoxSize, 3), a, b):
        H = L / N
        d = numpy.mod(numpy.arange(int(N)) * H - lo, L)
        out.append((d <= hi - lo).astype('f8'))
    return out


def restrict_to_box(field, a, b):
    """zero the cells of this rank's x slab of `field` (RealField) outside the box [a, b] (box_mask).  A window paint
    without interlacing is already zero there.  An interlaced paint is not: its second paint is shifted back by half a
    cell in Fourier space, which leaves band-limited tails on every cell; cut here, they cannot pair through the
    periodic wrap."""
    pm = field.pm
    mx, my, mz = (torch.as_tensor(m, dtype=field.value.dtype, device=field.value.device)
                  for m in box_mask(pm.Nmesh, pm.BoxSize, a, b))
    v = field.value.view(pm.x_n, int(pm.Nmesh[1]), int(pm.Nmesh[2]))
    v.mul_(mx[pm.x_start:pm.x_start + pm.x_n, None, None])
    v.mul_(my[None, :, None])
    v.mul_(mz[None, None, :])


def _fmt(v):
    return "[%s]" % ", ".join("%.6g" % x for x in v)


def pole_table(nnn, rrr, zeta, poles):
    """the (nb, nb) structured array of `.poles`: nnn_<l> per pole, then rrr_<l>, then zeta_<l>, in the order given"""
    nb = nnn.shape[-1]
    names = [('%s_%d' % (k, ell), 'f8') for k in ('nnn', 'rrr', 'zeta') for ell in poles]
    data = numpy.empty((nb, nb), dtype=names)
    for p, ell in enumerate(poles):
        data['nnn_%d' % ell] = nnn[p]
        data['rrr_%d' % ell] = rrr[p]
        data['zeta_%d' % ell] = zeta[p]
    return data


class ConvolvedFFT3PCF(object):
    r"""
    The edge-corrected multipoles :math:`\zeta_\ell(r_1, r_2)` of the isotropic three-point correlation function of a
    survey catalogue, measured on the mesh with FFTs (Slepian and Eisenstein, MNRAS 454, 4142 (2015) §4), on one or
    several GPUs.  Runs on construction.

    D and R are the data and randoms fields painted as :class:`FKPCatalogMesh` paints its species (mass u = w_c w_fkp
    Value, the mesh's window and interlacing, no compensation), then set to zero outside the window box: per axis
    [lo - (support / 2 + 1) H, hi + (support / 2 + 1) H] about the selected positions (lo / hi below).  Every cell a
    window paints lies inside it, so without interlacing this changes nothing; an interlaced paint shifts its second
    half back by half a cell in Fourier space, which leaves band-limited tails on every cell, and those are cut.  With
    alpha = data.W / randoms.W and V_c the cell
    volume, N = (D - alpha R) / V_c (the FKP field; no mean is subtracted) and Rf = alpha R / V_c.  With true
    (non-periodic) grid separations s = n H, r = sqrt((s_x^2 + s_y^2) + s_z^2), bin b holding e_b < r <= e_{b+1} (r = 0
    in no bin),

    .. math::

        \mathrm{nnn}_\ell(b_1, b_2) = \frac{2\ell + 1}{16\pi^2} \sum_x N(x) \sum_{s_1 \in b_1} \sum_{s_2 \in b_2}
            N(x + s_1)\, N(x + s_2)\, P_\ell(\hat u_1 \cdot \hat u_2)

    (s1 = s2 included), rrr_l the same with Rf, and zeta = :func:`~nbodykit_b200.algorithms.threeptcf.edge_correct`
    (nnn, rrr, poles).  No shot noise is subtracted.

    The FFT is periodic, so the constructor proves that no pair within max(edges) wraps: over the selected data and
    randoms, per axis, (hi - lo) + (support + 2) H + max(edges) < L and max(edges) <= L / 2, where lo / hi bound the
    positions relative to BoxCenter and support is the window's; otherwise it raises ValueError naming the BoxSize that
    passes.  The window box is (hi - lo) + (support + 2) H wide, so two of its cells within max(edges) of each other
    are never joined through the wrap, and the periodic FFT sums are the true-separation sums.  It also raises when
    no randoms are selected or their weights sum to zero.  The cost is 2 + 3 nbins sum_l (2l + 1) transforms, whatever
    the object count.

    Parameters
    ----------
    first : FKPCatalog, FKPCatalogMesh
        cast as ConvolvedFFTPower casts it; 'f4' / 'f8' meshes, and 'c8' / 'c16' meshes (whose real field is stored
        in the real-dtype mesh)
    poles : list of int
        every multipole from 0 to max(poles) <= 10, in any order (the edge correction couples them)
    edges : array_like
        radial bin edges, finite, strictly increasing, the first >= 0; at most 32 bins
    Nmesh : optional
        as for ConvolvedFFTPower

    When the bin fields of one (l, m) do not fit in free device memory (or NBK_BISPEC_RESIDENT caps them), the bins
    are processed in blocks, as in FFT3PCF; ``attrs['transforms']`` counts the transforms run.

    Attributes
    ----------
    poles : BinnedStatistic
        dims ``['r1', 'r2']``; fields ``nnn_<l>`` for every pole, then ``rrr_<l>``, then ``zeta_<l>``, in the order
        given (zeta is NaN where rrr_0 = 0)
    nsep : numpy.ndarray
        u8 per radial bin: the grid separations in the bin
    attrs : dict
        poles, edges, Nmesh, BoxSize, BoxCenter, alpha, data.W, randoms.W, transforms and tiles (the fraction of the
        Gram's 64-cell tiles that hold a nonzero weight, over both fields and all ranks)
    """
    logger = logging.getLogger('ConvolvedFFT3PCF')

    def __init__(self, first, poles, edges, Nmesh=None):
        poles = check_contiguous_poles(poles)
        e = _check_edges(edges)
        first = _cast_mesh(first, Nmesh=Nmesh)
        self.first = first
        self.comm = first.comm
        self.attrs = {}
        self.attrs['poles'] = poles
        self.attrs['edges'] = e
        self.attrs['Nmesh'] = numpy.array(first.attrs['Nmesh']).copy()
        self.attrs['BoxSize'] = numpy.asarray(first.attrs['BoxSize'], dtype='f8')
        self.attrs['BoxCenter'] = numpy.asarray(first.attrs['BoxCenter'], dtype='f8')
        self.attrs['mesh.resampler'] = first.resampler
        self.attrs['mesh.interlaced'] = first.interlaced
        lo, hi = numpy.full(3, numpy.inf), numpy.full(3, -numpy.inf)
        with stage("convfft3pcf_guard"):
            for name in ('data', 'randoms'):
                a, b = self._bounds(name)
                if name == 'randoms' and not (numpy.isfinite(a).all() and numpy.isfinite(b).all()):
                    raise ValueError("ConvolvedFFT3PCF: no randoms are selected; the edge correction needs their "
                                     "triplets")
                lo, hi = numpy.minimum(lo, a), numpy.maximum(hi, b)
            for name in ('data', 'randoms'):
                self.attrs[name + '.W'] = first.weighted_total(name)
        if not self.attrs['randoms.W'] > 0:
            raise ValueError("ConvolvedFFT3PCF: the selected randoms have a total weight of %r; alpha = data.W / "
                             "randoms.W needs it positive" % self.attrs['randoms.W'])
        self.support = FindResampler(first.resampler).support
        geometry_guard(lo, hi, self.attrs['Nmesh'], self.attrs['BoxSize'], self.support, float(e[-1]))
        self.window = window_box(lo, hi, self.attrs['BoxSize'] / self.attrs['Nmesh'], self.support)
        self.run()

    def _bounds(self, name):
        """(lo, hi) of the selected positions of species `name` relative to BoxCenter, over all ranks"""
        from ..base.catalog import ConstantColumn
        mesh = self.first
        cat = mesh.source[name]
        sel = cat[mesh.selection]
        sel = None if isinstance(sel, ConstantColumn) and bool(sel.value) else sel.compute()
        pos = mesh.RecenteredPosition(name)
        return get_data_bounds(pos.compute() if hasattr(pos, 'compute') else pos, self.comm, selection=sel)

    def run(self):
        mesh = self.first
        attrs = self.attrs
        poles = attrs['poles']
        e = numpy.asarray(attrs['edges'], dtype='f8')
        alpha = attrs['data.W'] / attrs['randoms.W']
        attrs['alpha'] = alpha
        with stage("convfft3pcf_paint"):
            N = mesh['data'].to_real_field(normalize=False)
            R = mesh['randoms'].to_real_field(normalize=False)
        with stage("convfft3pcf_fields"):
            pm = N.pm
            vc = float((pm.BoxSize / pm.Nmesh).prod())
            N.axpy(R, -alpha)
            N /= vc
            R *= alpha / vc
            # zero outside the window box (a no-op unless the mesh is interlaced), so that no pair wraps
            for f in (N, R):
                restrict_to_box(f, *self.window)
        with stage("fft3pcf_r2c"):
            Nhat = N.r2c()
            Rhat = R.r2c()
        with stage("convfft3pcf_tiles"):
            tN, tR = tile_list(N), tile_list(R)
            ntile = -(-int(numpy.prod(pm.real_shape)) // GRAM_TILE)
            listed = self.comm.allreduce(int(tN.numel()) + int(tR.numel()))
            total = self.comm.allreduce(2 * ntile)
        attrs['tiles'] = listed / total if total else 0.
        sums, n = bin_pass(pm, [(N, Nhat, tN), (R, Rhat, tR)], e, poles)
        del N, R, Nhat, Rhat
        nnn, rrr = sums
        attrs['transforms'] = 2 + n
        with stage("convfft3pcf_finish"):
            self.nsep = separation_counts(pm.Nmesh, pm.BoxSize, e)
            zeta = edge_correct(nnn, rrr, poles)
        self.poles = BinnedStatistic(['r1', 'r2'], [e, e], pole_table(nnn, rrr, zeta, poles))
        return self.poles

    def __getstate__(self):
        return dict(poles=self.poles.__getstate__(), nsep=self.nsep, attrs=self.attrs)

    def __setstate__(self, state):
        self.attrs = state['attrs']
        self.nsep = numpy.asarray(state['nsep']).astype('u8')
        self.poles = BinnedStatistic.from_state(state['poles'])

    def save(self, output):
        import json
        if self.comm.rank == 0:
            self.logger.info('saving ConvolvedFFT3PCF result to %s' % output)
            with open(output, 'w') as ff:
                json.dump(self.__getstate__(), ff, cls=JSONEncoder)

    @classmethod
    @CurrentMPIComm.enable
    def load(cls, output, comm=None):
        import json
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
