"""
FFT3PCF -- the multipoles of the isotropic three-point correlation function of a periodic box on the mesh, with FFTs
(the FFT form of the Slepian & Eisenstein estimator: MNRAS 454, 4142 (2015); MNRAS 455, L31 (2016)).  The reference
has no mesh 3PCF: this extends the package past it, with SimulationBox3PCF's conventions (DESIGN.md §4.16).

With delta = F - mean(F) on the mesh, grid separations s = n H (n_i in (-N_i/2, N_i/2], SimulationBox3PCF's periodic
wrap) and real orthonormal Y_lm, the addition theorem turns the triple sum into

    a_lm,b(x) = sum_{s in b} Y_lm(s / |s|) delta(x + s) = c2r(r2c(delta) conj(r2c(K_lm,b))) N_cells,  K_lm,b = Y_lm 1_b
    corr_l(b1, b2) = (1 / 4 pi) sum_m sum_x delta a_lm,b1 a_lm,b2

The kernel fields K and the weighted Gram sums are CUDA kernels (csrc/fft3pcf.cu); the product is nbk_cross_power and
the transforms are RealField.r2c / ComplexField.c2r.
"""
import logging

import numpy
import torch

from .._lib import check, darr, lib, stage
from ..binned_statistic import BinnedStatistic
from ..pmesh.pm import ComplexField, RealField, _ptr, _stream, _CODE
from .bispectrum import _resident_cap
from .fftpower import FFTBase
from .threeptcf import _check_edges, _check_poles, coefficient_table


# cells per tile of the Gram (F3_TILE of csrc/fft3pcf.cu): the unit of the tile lists of nbk_fft3pcf_gram_tiles
GRAM_TILE = 64


def transform_count(blocks, poles, sources=1):
    """the r2c and c2r transforms of one call on the bin blocks `blocks` (bin_blocks) with `sources` weighted fields
    (bin_pass): one r2c per field, then per (l, m) one r2c per kernel field built and one c2r per field -- block p is
    built once as the first of its pairs and once for each earlier block"""
    return sources + (1 + sources) * sum(2 * ell + 1 for ell in poles) * sum(len(b) * (1 + p)
                                                                           for p, b in enumerate(blocks))


def bin_blocks(nbins, cap):
    """the bins in blocks of resident fields: one block when all `cap` fields fit, else blocks of cap // 2 (two blocks
    are resident at once)"""
    bsz = nbins if cap >= nbins else max(cap // 2, 1)
    return [list(range(b, min(b + bsz, nbins))) for b in range(0, nbins, bsz)]


def separation_counts(Nmesh, BoxSize, edges):
    """nsep: the number of grid separations in each radial bin, u8 (host, exact: the kernel's float64 arithmetic)"""
    N = [int(v) for v in numpy.broadcast_to(Nmesh, 3)]
    L = numpy.broadcast_to(numpy.asarray(BoxSize, dtype='f8'), 3)
    e = numpy.asarray(edges, dtype='f8')
    nb = len(e) - 1
    rmax = float(e[-1])
    s = []
    for d in range(3):
        i = numpy.arange(N[d])
        n = numpy.where(2 * i <= N[d], i, i - N[d]).astype('f8')
        v = n * (L[d] / N[d])
        s.append(v[numpy.abs(v) <= rmax * (1 + 1e-9)])      # |s_d| <= r: no separation in a bin is left out
    sy, sz = s[1][:, None], s[2][None, :]
    syz = sy * sy
    zz = sz * sz
    counts = numpy.zeros(nb, dtype='u8')
    for sx in s[0]:
        r = numpy.sqrt((sx * sx + syz) + zz)
        b = numpy.searchsorted(e, r, side='left') - 1            # e_b < r <= e_{b+1}
        ok = (r > 0) & (b >= 0) & (b < nb)
        counts += numpy.bincount(b[ok], minlength=nb).astype('u8')
    return counts


def tile_list(w):
    """the indices (device int64) of the GRAM_TILE-cell tiles of the local field `w` (RealField) that hold a nonzero
    cell: the tiles nbk_fft3pcf_gram_tiles visits.  Its sum over them is the dense Gram's, as w = 0 on the others."""
    v = w.value.reshape(-1)
    pad = (-v.numel()) % GRAM_TILE
    if pad:
        v = torch.cat([v, v.new_zeros(pad)])
    return torch.nonzero((v.view(-1, GRAM_TILE) != 0).any(dim=1)).reshape(-1)


def bin_pass(pm, sources, edges, poles):
    """the Gram sums of FFT3PCF and ConvolvedFFT3PCF.  `sources` is a list of (w, what, tiles): a weight RealField w, the
    spectrum what (ComplexField) of the field the bin kernels are applied to, and None (the dense Gram) or w's
    tile_list (the listed Gram).  Per (l, m) and radial bin b the kernel field K = Y_lm 1_b is filled and transformed
    once; per source, c2r(what conj(K^) N_cells) = sum_{s in b} Y_lm(s) f(x + s) goes to that source's resident store
    (the last product is formed in K^'s own buffer, the others in scratch spectra), and one Gram per source and block
    pair accumulates sum_x w a_i b_j.  Bins that do not fit run in blocks (bin_blocks; the stores of every source count
    against free memory).  One all-reduce carries the packed float64 sums.

    Returns the (len(sources), len(poles), nb, nb) host array (1 / 4 pi) sum_m sum_x w a_lm,b1 a_lm,b2 (all ranks) and
    the number of transforms run (those of the spectra `what` not included)."""
    e = numpy.asarray(edges, dtype='f8')
    nb = len(e) - 1
    nsrc = len(sources)
    L = max(poles)
    T = darr(numpy.ascontiguousarray(coefficient_table(L)).ravel())
    code = _CODE[pm.typestr]
    tdt = torch.float64 if pm.typestr == 'f8' else torch.float32
    cdt = torch.complex128 if pm.typestr == 'f8' else torch.complex64
    dev = sources[0][0].value.device
    ncell = int(numpy.prod(pm.real_shape))
    ncells = int(numpy.prod(pm.Nmesh))

    # the kernel field, its spectrum, the scratch spectra, the transforms' work buffers and a margin stay free
    cslab = int(numpy.prod(pm.complex_shape))
    esz = torch.empty((), dtype=cdt).element_size()
    fsz = ncell * torch.empty((), dtype=tdt).element_size()
    reserve = (3 + nsrc) * cslab * esz + fsz + (256 << 20)
    cap = _resident_cap(nb, nsrc * fsz, reserve, pm.comm)
    blocks = bin_blocks(nb, cap)
    bsz = len(blocks[0])
    stores = [torch.empty((bsz if len(blocks) == 1 else 2 * bsz, ncell), dtype=tdt, device=dev) for _ in sources]
    K = RealField(pm)
    Khat = ComplexField(pm)
    prods = [ComplexField(pm) for _ in sources[:-1]] + [Khat]
    # one float64 accumulator per source, pole and block pair (p <= q), packed for the single all-reduce
    pairs = [(p, q) for p in range(len(blocks)) for q in range(p, len(blocks))]
    offs, o = {}, 0
    for pq in pairs:
        offs[pq] = o
        o += len(blocks[pq[0]]) * len(blocks[pq[1]])
    sums = torch.zeros((nsrc, len(poles), o), dtype=torch.float64, device=dev)
    g = lib()
    box = pm._box_c
    edges_c = darr(e)
    counted = [0]

    def build(bins, row0, ell, m):
        """a_lm,b of every source for the bins `bins` into store rows row0, row0 + 1, ..."""
        for q, b in enumerate(bins):
            with stage("fft3pcf_fill"):
                check(g.nbk_fft3pcf_kernel_fill(_ptr(K.value), code, pm._nmesh_c, box, pm.x_start, pm.x_n, edges_c,
                                                len(e), b, ell, m, 1, T, L, ncell, _stream()), "nbk_fft3pcf_kernel_fill")
            with stage("fft3pcf_r2c"):
                K.r2c(out=Khat)
            with stage("fft3pcf_product"):
                # what conj(K^) into the source's buffer, the last one into K^'s own (every element's inputs are read
                # before it is written), times N_cells: c2r of the product is then sum_s K(s) f(x + s)
                for (_, what, _), out in zip(sources, prods):
                    check(g.nbk_cross_power(_ptr(what.value), _ptr(Khat.value), _ptr(out.value), code,
                                            Khat.value.numel(), float(ncells), 0, _stream()), "nbk_cross_power")
            with stage("fft3pcf_c2r"):
                for out, store in zip(prods, stores):
                    out.c2r(out=RealField(pm, store[row0 + q].view(pm.real_shape)))
            counted[0] += 1 + nsrc

    def gram(p, pa, pb):
        """sum_x w a_i b_j of the resident blocks: pa from store row 0, pb (when another block) from row bsz"""
        A, B = blocks[pa], blocks[pb]
        rowb = 0 if pa == pb else bsz
        with stage("fft3pcf_gram"):
            for s, ((w, _, tiles), store) in enumerate(zip(sources, stores)):
                out = sums[s, p, offs[(pa, pb)]:]
                if tiles is None:
                    check(g.nbk_fft3pcf_gram(_ptr(w.value), _ptr(store[0]), ncell, len(A), _ptr(store[rowb]), ncell,
                                             len(B), code, ncell, _ptr(out), _stream()), "nbk_fft3pcf_gram")
                else:
                    check(g.nbk_fft3pcf_gram_tiles(_ptr(w.value), _ptr(store[0]), ncell, len(A), _ptr(store[rowb]),
                                                   ncell, len(B), code, ncell, _ptr(tiles), tiles.numel(), _ptr(out),
                                                   _stream()), "nbk_fft3pcf_gram_tiles")

    for p, ell in enumerate(poles):
        for m in range(-ell, ell + 1):
            for pa in range(len(blocks)):
                build(blocks[pa], 0, ell, m)
                gram(p, pa, pa)
                for pb in range(pa + 1, len(blocks)):
                    build(blocks[pb], bsz, ell, m)
                    gram(p, pa, pb)
    del stores, K, Khat, prods
    with stage("fft3pcf_allreduce"):
        if pm.comm.size > 1:
            pm.comm.allreduce_tensor(sums)
    host = sums.cpu().numpy()
    corr = numpy.zeros((nsrc, len(poles), nb, nb))
    for (pa, pb) in pairs:
        A, B = blocks[pa], blocks[pb]
        part = host[:, :, offs[(pa, pb)]:offs[(pa, pb)] + len(A) * len(B)].reshape(nsrc, len(poles), len(A), len(B))
        corr[:, :, A[0]:A[-1] + 1, B[0]:B[-1] + 1] = part
    iu = numpy.triu_indices(nb, 1)
    corr[:, :, iu[1], iu[0]] = corr[:, :, iu[0], iu[1]]             # the Gram adds i <= j of a block with itself
    corr /= 4 * numpy.pi
    return corr, counted[0]


class FFT3PCF(FFTBase):
    r"""
    The multipoles :math:`\zeta_\ell(r_1, r_2)` of the isotropic three-point correlation function of a periodic box,
    measured on the mesh with FFTs (Slepian and Eisenstein, MNRAS 455, L31 (2016)), on one or several GPUs.  Runs on
    construction.

    The field is F = ``first.compute(mode='real')`` and delta = F - mean(F).  The mesh nodes play the objects of
    :class:`SimulationBox3PCF` and delta their weights: with grid separations s = (n_x H_x, n_y H_y, n_z H_z),
    H_i = L_i / N_i, n_i in (-N_i/2, N_i/2], r = sqrt((s_x^2 + s_y^2) + s_z^2) in float64 and bin b holding
    e_b < r <= e_{b+1} (r = 0 in no bin),

    .. math::

        \mathrm{corr}_\ell(b_1, b_2) = \frac{2\ell + 1}{16\pi^2} \sum_x \delta(x) \sum_{s_1 \in b_1} \sum_{s_2 \in b_2}
            \delta(x + s_1)\, \delta(x + s_2)\, P_\ell(\hat u_1 \cdot \hat u_2)

    (periodic shifts, s1 = s2 included) and :math:`\zeta_\ell = 16\pi^2 \mathrm{corr}_\ell / (N_{cells}\,
    n_{sep}[b_1]\, n_{sep}[b_2])`, the Legendre coefficient of <delta delta delta> over the bin pair.  No shot noise is
    subtracted.  The cost is 1 + 2 nbins sum_l (2l + 1) transforms, whatever the object count.

    Parameters
    ----------
    first : CatalogSource, MeshSource
        the source; a catalogue is painted as FFTPower paints it (f8, compensated)
    poles : list of int
        distinct multipoles, 0 .. :func:`~nbodykit_b200.algorithms.threeptcf.max_ell` (10); odd ell allowed
    edges : array_like
        radial bin edges, finite, strictly increasing, the first >= 0; at most
        :func:`~nbodykit_b200.algorithms.threeptcf.max_bins` (32) bins; max(edges) <= half the smallest side
    Nmesh, BoxSize : optional
        as for FFTPower

    When the bin fields of one (l, m) do not fit in free device memory (or NBK_BISPEC_RESIDENT caps them), the bins
    are processed in blocks and fields are rebuilt per block pair; ``attrs['transforms']`` counts the transforms run.

    Attributes
    ----------
    poles : BinnedStatistic
        dims ``['r1', 'r2']``; fields ``corr_<l>`` for every pole, then ``zeta_<l>`` for every pole, in the order given
        (zeta is NaN for a bin without separations)
    nsep : numpy.ndarray
        u8 per radial bin: the grid separations in the bin
    attrs : dict
        poles, edges, Nmesh, BoxSize, transforms, N1, shotnoise (and FFTBase's Lx, Ly, Lz, volume)
    """
    logger = logging.getLogger('FFT3PCF')

    def __init__(self, first, poles, edges, Nmesh=None, BoxSize=None):
        poles = _check_poles(poles)
        e = _check_edges(edges)
        FFTBase.__init__(self, first, None, Nmesh, BoxSize)
        if e[-1] > 0.5 * numpy.asarray(self.attrs['BoxSize'], dtype='f8').min():
            raise ValueError("periodic 3PCF cannot be computed for Rmax > BoxSize/2")
        self.attrs['poles'] = poles
        self.attrs['edges'] = e
        self.run()

    def run(self):
        attrs = self.attrs
        poles = attrs['poles']
        e = numpy.asarray(attrs['edges'], dtype='f8')
        with stage("fft3pcf_paint"):
            F = self.first.compute(mode='real', Nmesh=attrs['Nmesh'])
        attrs['N1'] = F.attrs.get('N', 0)
        attrs['shotnoise'] = F.attrs.get('shotnoise', 0)
        pm = F.pm
        if pm.cplx:
            # a complex-typed mesh stores its real field as a real array: the real-dtype mesh takes it as it is
            pm = pm.reshape(dtype=pm.typestr)
            F = RealField(pm, F.value)
        ncells = int(numpy.prod(pm.Nmesh))
        with stage("fft3pcf_mean"):
            mean = F.csum() / ncells                               # the one all-reduce of the mean
        delta = RealField(pm)
        with stage("fft3pcf_delta"):
            delta[...] = -mean
            delta.axpy(F, 1.0)
        del F
        with stage("fft3pcf_r2c"):
            dhat = delta.r2c()
        corr, n = bin_pass(pm, [(delta, dhat, None)], e, poles)
        del dhat, delta
        self.nsep = separation_counts(pm.Nmesh, pm.BoxSize, e)
        attrs['transforms'] = 1 + n
        self.poles = BinnedStatistic(['r1', 'r2'], [e, e], pole_table(corr[0], self.nsep, ncells, poles))
        return self.poles

    def __getstate__(self):
        return {'poles': self.poles.data, 'nsep': self.nsep, 'attrs': self.attrs}

    def __setstate__(self, state):
        self.attrs = state['attrs']
        self.nsep = numpy.asarray(state['nsep']).astype('u8')
        self.poles = BinnedStatistic(['r1', 'r2'], [numpy.asarray(self.attrs['edges'])] * 2, state['poles'])


def pole_table(corr, nsep, ncells, poles):
    """the (nb, nb) structured array of `.poles`: corr_<l> per pole, then zeta_<l> = 16 pi^2 corr_l / (N_cells nsep[b1]
    nsep[b2]) per pole (NaN where a bin holds no separation)"""
    nb = corr.shape[-1]
    data = numpy.empty((nb, nb), dtype=[('corr_%d' % ell, 'f8') for ell in poles] + [('zeta_%d' % ell, 'f8')
                                                                                   for ell in poles])
    nn = numpy.outer(numpy.asarray(nsep, dtype='f8'), numpy.asarray(nsep, dtype='f8'))
    for p, ell in enumerate(poles):
        data['corr_%d' % ell] = corr[p]
        with numpy.errstate(invalid='ignore', divide='ignore'):
            data['zeta_%d' % ell] = numpy.where(nn > 0, 16 * numpy.pi ** 2 * corr[p] / (float(ncells) * nn), numpy.nan)
    return data
