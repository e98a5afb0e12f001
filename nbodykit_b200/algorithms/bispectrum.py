"""
FFTBispectrum -- the bispectrum B(k1, k2, k3) of a periodic box with the FFT estimator (Scoccimarro 2015,
arXiv:1506.02729 §III; Sefusatti et al. 2016, arXiv:1512.07295).  The reference has no bispectrum: this extends the
package past it, with FFTPower's conventions (DESIGN.md §4.14).

Per k shell S_i, I_i = c2r(c 1_{S_i}) (mesh precision) and J_i = c2r(1_{S_i}) (float64) are real x-slab fields; for every
sorted shell triple i <= j <= l that can close,

    T_ijl = sum_x J_i J_j J_l / N^3        (ordered triplets q_a in S_a with q1 + q2 + q3 = 0 modulo the grid)
    B_ijl = V^2 sum_x I_i I_j I_l / sum_x J_i J_j J_l

The shell fill and the triple sum are CUDA kernels (csrc/bispectrum.cu); the transforms are ComplexField.c2r.
"""
import logging
import os

import numpy
import torch

from .. import _lib
from .._lib import check, lib, stage
from ..binned_statistic import BinnedStatistic
from ..pmesh.pm import ComplexField, RealField, _ptr, _stream, _CODE
from .fftpower import FFTBase, project_to_basis_device

# the most shells one fill call writes into its scratch slabs (each the size of the complex field)
_FILL_CHUNK = 4


def max_shells():
    """the largest number of k shells the kernels take"""
    return int(lib().nbk_bispec_max_shells())


def shell_edges(Nmesh, BoxSize, dk=None, kmin=0., kmax=None):
    """the shell edges ``numpy.arange(kmin, kmax, dk)`` with FFTPower's defaults (dk = 2 pi / min(L),
    kmax = pi min(N) / max(L) + dk / 2); raises ValueError for dk = 0 (unique edges), a negative kmin, no shell at all,
    or more than :func:`max_shells` shells"""
    Nmesh = numpy.asarray(Nmesh) * numpy.ones(3, dtype='i8')
    BoxSize = numpy.asarray(BoxSize, dtype='f8') * numpy.ones(3)
    if dk is None:
        dk = 2 * numpy.pi / BoxSize.min()
    if dk == 0:
        raise ValueError("FFTBispectrum needs uniform shells (dk > 0); unique edges (dk = 0) are not supported")
    if not dk > 0:
        raise ValueError("FFTBispectrum needs dk > 0, got %r" % dk)
    if kmin < 0:
        raise ValueError("FFTBispectrum needs kmin >= 0, got %r" % kmin)
    if kmax is None:
        kmax = numpy.pi * Nmesh.min() / BoxSize.max() + dk / 2
    kedges = numpy.arange(kmin, kmax, dk)
    nshell = len(kedges) - 1
    if nshell < 1:
        raise ValueError("FFTBispectrum: no k shell between kmin = %r and kmax = %r with dk = %r" % (kmin, kmax, dk))
    if nshell > max_shells():
        raise ValueError("FFTBispectrum: %d k shells, more than the maximum of %d (max_shells()); raise dk or lower kmax"
                         % (nshell, max_shells()))
    return kedges


def shell_triples(kedges):
    """the sorted shell triples i <= j <= l that are evaluated, (ntri, 3) int32 in lexicographic order: those with
    kedges[l] < kedges[i + 1] + kedges[j + 1], the only ones that can hold a closed triangle of |k|"""
    e = numpy.asarray(kedges, dtype='f8')
    n = len(e) - 1
    out = [(i, j, l) for i in range(n) for j in range(i, n) for l in range(j, n) if e[l] < e[i + 1] + e[j + 1]]
    return numpy.array(out, dtype='i4').reshape(-1, 3)


def bispectrum_table(kedges, kmean, triples, S, Tsum, volume, Ncells):
    """the (n, n, n) structured array of `.bispec` from the triple sums: S = sum_x I I I and Tsum = sum_x J J J per row
    of `triples`.  Every index permutation of a triple is filled; triples not evaluated report triangles = 0, B = NaN."""
    n = len(kedges) - 1
    data = numpy.zeros((n, n, n), dtype=[('k1', 'f8'), ('k2', 'f8'), ('k3', 'f8'), ('B', 'f8'), ('triangles', 'i8')])
    kmean = numpy.asarray(kmean, dtype='f8')
    data['k1'] = kmean[:, None, None]
    data['k2'] = kmean[None, :, None]
    data['k3'] = kmean[None, None, :]
    data['B'] = numpy.nan
    S = numpy.asarray(S, dtype='f8')
    Tsum = numpy.asarray(Tsum, dtype='f8')
    count = numpy.rint(Tsum / float(Ncells)).astype('i8')
    with numpy.errstate(invalid='ignore', divide='ignore'):
        B = numpy.where(count > 0, volume ** 2 * S / Tsum, numpy.nan)
    for (i, j, l), t, b in zip(numpy.asarray(triples).reshape(-1, 3), count, B):
        for p in {(i, j, l), (i, l, j), (j, i, l), (j, l, i), (l, i, j), (l, j, i)}:
            data['triangles'][p] = t
            data['B'][p] = b
    return data


def _resident_cap(nshell, field_bytes, reserve_bytes, comm):
    """how many real shell fields of one pass stay resident: what free device memory holds after `reserve_bytes`,
    capped by NBK_BISPEC_RESIDENT; the same on every rank (the transforms are collective)"""
    free, _ = torch.cuda.mem_get_info()
    free += torch.cuda.memory_reserved() - torch.cuda.memory_allocated()     # cached by torch, free to reuse
    cap = max(int((free - reserve_bytes) // field_bytes), 0)
    env = os.environ.get("NBK_BISPEC_RESIDENT")
    if env:
        cap = min(cap, int(env))
    cap = int(comm.allreduce(min(cap, nshell), op="min"))
    if cap < min(3, nshell):
        raise MemoryError("FFTBispectrum: room for only %d resident shell fields, at least %d are needed "
                          "(NBK_BISPEC_RESIDENT=%s)" % (cap, min(3, nshell), env))
    return cap


class FFTBispectrum(FFTBase):
    """
    Bispectrum of one source in a periodic box with the FFT estimator (Scoccimarro 2015, §III): for k shells
    ``kedges = numpy.arange(kmin, kmax, dk)`` (FFTPower's defaults) and every shell triple (k1, k2, k3)

        B = V^2 <delta(q1) delta(q2) delta(q3)>   over q_a in shell a with q1 + q2 + q3 = 0 modulo the grid

    with delta = ``compute(mode='complex')`` (forward transform normalised by 1/N^3).  A mode belongs to shell i when
    FFTPower puts it in k bin i (float32 coordinates); the k = 0 mode belongs to no shell.  Only shell triples with
    ``kedges[l] < kedges[i+1] + kedges[j+1]`` (sorted i <= j <= l) are evaluated; the others report ``triangles = 0`` and
    ``B = NaN``.  Closure is modulo the grid, as in every FFT estimator: shells above 2/3 of the Nyquist wavenumber
    include wrapped (aliased) triangles.

    Shot noise is NOT subtracted (as in FFTPower).  For a Poisson sample of unit weights it is
    ``S (P1 + P2 + P3) - 2 S^2`` with S = ``attrs['shotnoise']`` and P_a the measured power of shell a (``.power``).

    At most :func:`max_shells` shells.  When the shell fields of a pass do not fit in free device memory (or
    NBK_BISPEC_RESIDENT caps them), the shells are processed in blocks and fields are rebuilt per block triple;
    ``attrs['transforms']`` counts the c2r transforms run.

    Results, computed in __init__: ``.bispec`` (BinnedStatistic, dims k1, k2, k3; fields k1, k2, k3 -- the shells'
    mean |k| --, B, triangles), ``.power`` (the 1-D power spectrum on the same shells, as FFTPower(mode='1d') gives it)
    and ``.attrs``.
    """
    logger = logging.getLogger('FFTBispectrum')

    def __init__(self, first, Nmesh=None, BoxSize=None, dk=None, kmin=0., kmax=None):
        FFTBase.__init__(self, first, None, Nmesh, BoxSize)
        if dk is None:
            dk = 2 * numpy.pi / self.attrs['BoxSize'].min()
        self.attrs['dk'] = dk
        self.attrs['kmin'] = kmin
        self.attrs['kmax'] = kmax
        self.run()

    def run(self):
        kedges = shell_edges(self.attrs['Nmesh'], self.attrs['BoxSize'], self.attrs['dk'], self.attrs['kmin'],
                             self.attrs['kmax'])
        triples = shell_triples(kedges)
        with stage("H:compute_fields"):
            c = self.first.compute(mode='complex', Nmesh=self.attrs['Nmesh'])
        attrs = dict(self.attrs)
        attrs['N1'] = c.attrs.get('N', 0)
        attrs['shotnoise'] = c.attrs.get('shotnoise', 0)
        if not c.compressed:
            c = _compress(c)
        pm = c.pm
        V = float(self.attrs['BoxSize'].prod())

        # the 1-D power on the same shells, through FFTPower's binning
        result, _ = project_to_basis_device(c, [kedges, numpy.array([-1., 1.])], is_p3d=False, volume=V, need_mu=False)
        xmean, _, pk, modes = [numpy.asarray(r)[:, 0] for r in result]
        power = numpy.empty(len(kedges) - 1, dtype=[('k', 'f8'), ('power', pk.dtype.str), ('modes', modes.dtype.str)])
        power['k'], power['power'], power['modes'] = xmean, pk, modes
        kmean = xmean.copy()
        if kedges[0] == 0 and modes[0] > 1:
            # FFTPower counts the k = 0 mode in the first bin; the shells leave it out
            kmean[0] = xmean[0] * modes[0] / (modes[0] - 1)

        transforms = 0
        sums = []
        for indicator in (False, True):
            s, n = self._pass(c, kedges, triples, indicator)
            sums.append(s)
            transforms += n
        packed = torch.cat(sums)
        with stage("bispec_allreduce"):
            if pm.comm.size > 1:
                pm.comm.allreduce_tensor(packed)
        host = packed.cpu().numpy()
        ntri = len(triples)
        data = bispectrum_table(kedges, kmean, triples, host[:ntri], host[ntri:], V, int(numpy.prod(pm.Nmesh)))
        attrs['transforms'] = transforms
        self.attrs.update(attrs)
        self.power = BinnedStatistic(['k'], [kedges], power, fields_to_sum=['modes'], **self.attrs)
        self.bispec = BinnedStatistic(['k1', 'k2', 'k3'], [kedges] * 3, data, **self.attrs)
        return self.bispec

    def _pass(self, c, kedges, triples, indicator):
        """sum_x f_i f_j f_l for every triple, f = I (c 1_S in the mesh precision) or, indicator=True, J (1_S in float64).
        Returns the (ntri,) float64 device sums of this rank's x slab and the number of c2r transforms run."""
        pm = c.pm if not indicator else c.pm.reshape(dtype='f8')
        nshell = len(kedges) - 1
        ntri = len(triples)
        dev = c.value.device
        code = _CODE[pm.typestr]
        tdt = torch.float64 if pm.typestr == 'f8' else torch.float32
        cdt = torch.complex128 if pm.typestr == 'f8' else torch.complex64
        ncell = int(numpy.prod(pm.real_shape))
        cslab = int(numpy.prod(pm.complex_shape))
        fill_n = min(_FILL_CHUNK, nshell)
        # the fill scratch, the transform's work buffers and a margin stay free
        reserve = (fill_n + 4) * cslab * torch.empty((), dtype=cdt).element_size() + (256 << 20)
        cap = _resident_cap(nshell, ncell * torch.empty((), dtype=tdt).element_size(), reserve, pm.comm)
        # shell blocks: everything at once, or blocks of cap // 3 so that any three of them are resident together
        bsz = nshell if cap >= nshell else cap // 3
        blk = numpy.arange(nshell) // bsz
        key = blk[triples]                                    # (ntri, 3), non-decreasing along a row
        order = numpy.lexsort((key[:, 2], key[:, 1], key[:, 0])) if ntri else numpy.zeros(0, dtype='i8')
        store = torch.empty((min(cap, nshell), ncell), dtype=tdt, device=dev)
        scratch = torch.empty((fill_n,) + tuple(pm.complex_shape), dtype=cdt, device=dev)
        out = torch.zeros(ntri, dtype=torch.float64, device=dev)
        tr, start, count = c._slab()
        k2edges = _lib.darr((numpy.asarray(kedges) ** 2).astype('f8'))
        slot_of = {}                                          # resident shell -> row of `store`
        transforms = 0
        g0 = 0
        while g0 < ntri:
            g1 = g0
            while g1 < ntri and (key[order[g1]] == key[order[g0]]).all():
                g1 += 1
            rows = order[g0:g1]
            need = sorted(set(triples[rows].reshape(-1).tolist()))
            for s in [s for s in slot_of if s not in need]:
                del slot_of[s]
            free = sorted(set(range(store.shape[0])) - set(slot_of.values()))
            missing = [s for s in need if s not in slot_of]
            for s in missing:
                slot_of[s] = free.pop(0)
            # contiguous runs of missing shells, each filled in chunks of at most fill_n shells by one read of c
            runs = []
            for s in missing:
                if runs and runs[-1][-1] == s - 1 and len(runs[-1]) < fill_n:
                    runs[-1].append(s)
                else:
                    runs.append([s])
            for run in runs:
                with stage("bispec_fill"):
                    check(lib().nbk_bispec_fill(_ptr(c.value), _CODE[c.pm.typestr] if not indicator else code, pm._nmesh_c,
                                                pm._box_c, tr, start, count, k2edges, len(kedges), run[0], len(run),
                                                1 if indicator else 0, _ptr(scratch), cslab, _stream()), "nbk_bispec_fill")
                for q, s in enumerate(run):
                    with stage("bispec_c2r"):
                        ComplexField(pm, scratch[q]).c2r(out=RealField(pm, store[slot_of[s]].view(pm.real_shape)))
                    transforms += 1
            slots = numpy.vectorize(slot_of.get, otypes=['i4'])(triples[rows]) if len(rows) else None
            tri_dev = torch.from_numpy(numpy.ascontiguousarray(slots, dtype='i4')).to(dev)
            part = torch.zeros(len(rows), dtype=torch.float64, device=dev)
            with stage("bispec_triple_sum"):
                check(lib().nbk_bispec_triple_sum(_ptr(store), code, ncell, store.shape[0], ncell, _ptr(tri_dev), len(rows),
                                                  _ptr(part), _stream()), "nbk_bispec_triple_sum")
            out[torch.from_numpy(rows).to(dev)] = part
            g0 = g1
        del store, scratch
        return out, transforms

    def __getstate__(self):
        return dict(bispec=self.bispec.__getstate__(), power=self.power.__getstate__(), attrs=self.attrs)

    def __setstate__(self, state):
        self.attrs = state['attrs']
        self.bispec = BinnedStatistic.from_state(state['bispec'])
        self.power = BinnedStatistic.from_state(state['power'])


def _compress(c):
    """the Hermitian-compressed half of a complex-dtype mesh's full spectrum (one GPU), on the real-dtype mesh"""
    pm = c.pm
    Nx, Ny, Nz = [int(v) for v in pm.Nmesh]
    pmr = pm.reshape(dtype=pm.typestr)
    half = ComplexField(pmr)
    check(lib().nbk_hermitian_compress(_ptr(c.value), _ptr(half.value), _CODE[pm.typestr], Nx * Ny, Nz, _stream()),
          "nbk_hermitian_compress")
    half.attrs = dict(c.attrs)
    return half
