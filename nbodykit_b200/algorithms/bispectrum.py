"""
FFTBispectrum -- the bispectrum B(k1, k2, k3) of a periodic box with the FFT estimator (Scoccimarro 2015,
arXiv:1506.02729 §III; Sefusatti et al. 2016, arXiv:1512.07295).  The reference has no bispectrum: this extends the
package past it, with FFTPower's conventions (DESIGN.md §4.14).

Per k shell S_i, I_i = c2r(c 1_{S_i}) (mesh precision) and J_i = c2r(1_{S_i}) (float64) are real x-slab fields; for every
sorted shell triple i <= j <= l that can close,

    T_ijl = sum_x J_i J_j J_l / N^3        (ordered triplets q_a in S_a with q1 + q2 + q3 = 0 modulo the grid)
    B_ijl = V^2 sum_x I_i I_j I_l / sum_x J_i J_j J_l

Multipoles about a global line of sight (Scoccimarro 2015 §III): per even ell > 0 and shell a, W^ell_a = c2r(c L_ell(mu)
1_{S_a}) weights the first wavevector, and for every ordered row (a, b, c), b <= c, of an evaluated triple

    B_ell[a, b, c] = (2 ell + 1) V^2 sum_x W^ell_a I_b I_c / sum_x J_a J_b J_c

The shell fills and the triple sum are CUDA kernels (csrc/bispectrum.cu); the transforms are ComplexField.c2r.
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
# the largest multipole: even ell in [0, _MAX_ELL]
_MAX_ELL = 8


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


def check_poles(poles, los):
    """the validated multipole list (ints) for FFTBispectrum; raises ValueError, before any device work, for a
    line of sight that is not a unit 3-vector (FFTPower's rule), odd ell, ell outside [0, 8] or a repeated ell"""
    if numpy.isscalar(los) or len(los) != 3:
        raise ValueError("line-of-sight ``los`` should be vector with length 3")
    if not numpy.allclose(numpy.einsum('i,i', los, los), 1.0, rtol=1e-5):
        raise ValueError("line-of-sight ``los`` must be a unit vector")
    poles = [] if poles is None else list(poles)
    for ell in poles:
        if numpy.ndim(ell) != 0 or int(ell) != ell or not 0 <= ell <= _MAX_ELL:
            raise ValueError("FFTBispectrum: multipole %r; poles must be even integers 0 <= ell <= %d"
                             % (ell, _MAX_ELL))
        if ell % 2:
            raise ValueError("FFTBispectrum: odd multipole ell = %d; with a global line of sight an odd ell gives an "
                             "imaginary statistic, which the c2r of a Hermitian half spectrum cannot represent" % ell)
    if len(set(poles)) != len(poles):
        raise ValueError("FFTBispectrum: repeated multipole in poles = %r" % (poles,))
    return [int(ell) for ell in poles]


def pole_triples(kedges):
    """the weighted rows (a, b, c), b <= c, of the multipoles, (nrow, 3) int32: for every evaluated sorted triple
    (shell_triples order) one row per distinct shell a in it, ascending -- 3 rows for a scalene triple, 2 for an
    isosceles one, 1 for an equilateral one.  The Legendre weight sits on shell a."""
    rows = []
    for t in shell_triples(kedges).tolist():
        for a in sorted(set(t)):
            rest = list(t)
            rest.remove(a)
            rows.append([a] + rest)
    return numpy.array(rows, dtype='i4').reshape(-1, 3)


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


def poles_table(bispec, triples, rows, W, Tsum, volume, poles):
    """the (n, n, n) structured array of `.poles` from `.bispec`'s data: k1, k2, k3 and triangles as there, B_0 = its B;
    for ell > 0, W[ell] = sum_x W^ell_a I_b I_c per row (a, b, c) of `rows` (pole_triples) and Tsum = sum_x J J J per
    sorted triple of `triples` give B_ell[a, b, c] = B_ell[a, c, b] = (2 ell + 1) V^2 W / Tsum.  Entries whose sorted
    triple is not evaluated (or holds no triangle) report NaN."""
    shape = bispec.shape
    data = numpy.zeros(shape, dtype=[('k1', 'f8'), ('k2', 'f8'), ('k3', 'f8')] + [('B_%d' % ell, 'f8') for ell in poles]
                       + [('triangles', 'i8')])
    for f in ('k1', 'k2', 'k3', 'triangles'):
        data[f] = bispec[f]
    index = {tuple(t): q for q, t in enumerate(numpy.asarray(triples).reshape(-1, 3).tolist())}
    rows = numpy.asarray(rows).reshape(-1, 3)
    tri = numpy.array([index[tuple(sorted(r))] for r in rows.tolist()], dtype='i8')
    Tsum = numpy.asarray(Tsum, dtype='f8')[tri]
    count = bispec['triangles'][rows[:, 0], rows[:, 1], rows[:, 2]] if len(rows) else numpy.zeros(0, dtype='i8')
    for ell in poles:
        if ell == 0:
            data['B_0'] = bispec['B']
            continue
        with numpy.errstate(invalid='ignore', divide='ignore'):
            B = numpy.where(count > 0, (2 * ell + 1) * volume ** 2 * numpy.asarray(W[ell], dtype='f8') / Tsum, numpy.nan)
        col = numpy.full(shape, numpy.nan)
        col[rows[:, 0], rows[:, 1], rows[:, 2]] = B
        col[rows[:, 0], rows[:, 2], rows[:, 1]] = B
        data['B_%d' % ell] = col
    return data


def _resident_cap(nshell, field_bytes, reserve_bytes, comm):
    """how many real shell fields of one pass stay resident: what free device memory holds after `reserve_bytes`,
    capped by NBK_BISPEC_RESIDENT and by the max_shells() fields the triple sum stages; the same on every rank (the
    transforms are collective).  `nshell` is the number of fields of the pass."""
    free, _ = torch.cuda.mem_get_info()
    free += torch.cuda.memory_reserved() - torch.cuda.memory_allocated()     # cached by torch, free to reuse
    cap = max(int((free - reserve_bytes) // field_bytes), 0)
    env = os.environ.get("NBK_BISPEC_RESIDENT")
    if env:
        cap = min(cap, int(env))
    cap = int(comm.allreduce(min(cap, nshell, max_shells()), op="min"))
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

    Multipoles about the line of sight ``los`` (a unit 3-vector, as in FFTPower), for the even ``poles``
    0 <= ell <= 8 (odd ell are imaginary for a global line of sight and raise ValueError):

        B_ell[a, b, c] = (2 ell + 1) V^2 sum_x W^ell_a I_b I_c / sum_x J_a J_b J_c,   W^ell_a = c2r(c L_ell(mu) 1_{S_a})

    with the Legendre weight on the first wavevector k1 (shell a), so B_ell is symmetric in (b, c) only.  mu = q.los / |q|
    is formed in float32 as FFTPower forms it, L_ell in float64.  B_0 is ``.bispec['B']``; entries whose sorted triple is
    not evaluated report NaN.  Shot noise is NOT subtracted from B_ell either.  Each ell > 0 adds one c2r per shell.

    Results, computed in __init__: ``.bispec`` (BinnedStatistic, dims k1, k2, k3; fields k1, k2, k3 -- the shells'
    mean |k| --, B, triangles), ``.power`` (the 1-D power spectrum on the same shells, as FFTPower(mode='1d') gives it),
    ``.poles`` (with poles: BinnedStatistic with the same dims and fields k1, k2, k3, B_<ell> per requested ell,
    triangles; without: None) and ``.attrs``.
    """
    logger = logging.getLogger('FFTBispectrum')

    def __init__(self, first, Nmesh=None, BoxSize=None, dk=None, kmin=0., kmax=None, poles=[], los=[0, 0, 1]):
        poles = check_poles(poles, los)
        FFTBase.__init__(self, first, None, Nmesh, BoxSize)
        if dk is None:
            dk = 2 * numpy.pi / self.attrs['BoxSize'].min()
        self.attrs['dk'] = dk
        self.attrs['kmin'] = kmin
        self.attrs['kmax'] = kmax
        self.attrs['poles'] = poles
        self.attrs['los'] = los
        self.run()

    def run(self):
        kedges = shell_edges(self.attrs['Nmesh'], self.attrs['BoxSize'], self.attrs['dk'], self.attrs['kmin'],
                             self.attrs['kmax'])
        triples = shell_triples(kedges)
        nshell = len(kedges) - 1
        ells = sorted(ell for ell in self.attrs['poles'] if ell > 0)     # the weighted field families 1, 2, ...
        prows = pole_triples(kedges) if ells else numpy.zeros((0, 3), dtype='i4')
        # rows of the I pass over field ids family * nshell + shell: the sorted triples, then per ell > 0 the weighted
        # rows with their first field in that family
        rows = numpy.concatenate([triples] + [prows + numpy.array([(q + 1) * nshell, 0, 0], dtype='i4')
                                              for q in range(len(ells))])
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
            # the J pass needs only the family-0 fields: its store, residency and blocks are those of the plain call
            s, n = (self._pass(c, kedges, triples, True) if indicator else self._pass(c, kedges, rows, False, ells))
            sums.append(s)
            transforms += n
        packed = torch.cat(sums)
        with stage("bispec_allreduce"):
            if pm.comm.size > 1:
                pm.comm.allreduce_tensor(packed)
        host = packed.cpu().numpy()
        ntri, nrow = len(triples), len(rows)
        Tsum = host[nrow:]
        data = bispectrum_table(kedges, kmean, triples, host[:ntri], Tsum, V, int(numpy.prod(pm.Nmesh)))
        attrs['transforms'] = transforms
        self.attrs.update(attrs)
        self.power = BinnedStatistic(['k'], [kedges], power, fields_to_sum=['modes'], **self.attrs)
        self.bispec = BinnedStatistic(['k1', 'k2', 'k3'], [kedges] * 3, data, **self.attrs)
        self.poles = None
        if self.attrs['poles']:
            W = {ell: host[ntri + q * len(prows):ntri + (q + 1) * len(prows)] for q, ell in enumerate(ells)}
            pdata = poles_table(data, triples, prows, W, Tsum, V, self.attrs['poles'])
            self.poles = BinnedStatistic(['k1', 'k2', 'k3'], [kedges] * 3, pdata, **self.attrs)
        return self.bispec

    def _pass(self, c, kedges, triples, indicator, ells=()):
        """sum_x f_a f_b f_c for every row of `triples` (shell_pass), the weighted families those of `ells` about
        attrs['los']"""
        return shell_pass(c, kedges, triples, indicator, ells, los=self.attrs['los'])

    def __getstate__(self):
        return dict(bispec=self.bispec.__getstate__(), power=self.power.__getstate__(),
                    poles=self.poles.__getstate__() if getattr(self, 'poles', None) is not None else None,
                    attrs=self.attrs)

    def __setstate__(self, state):
        self.attrs = state['attrs']
        self.bispec = BinnedStatistic.from_state(state['bispec'])
        self.power = BinnedStatistic.from_state(state['power'])
        self.poles = None
        if state.get('poles') is not None:                   # results saved before multipoles have no 'poles'
            self.poles = BinnedStatistic.from_state(state['poles'])


def shell_pass(c, kedges, triples, indicator, ells=(), los=None, sources=()):
    """sum_x f_a f_b f_c for every row of `triples`, over the fields f = (family, shell) with field id
    family * nshell + shell: family 0 is I (c 1_S in the mesh precision) or, indicator=True, J (1_S in float64);
    family q > 0 is W^ell = c L_ell(mu) 1_S in the mesh precision, ell = ells[q - 1], mu about the unit 3-vector `los`.
    With `sources` instead of `ells`, family q > 0 is filled from its own compressed field(s) on c's mesh and layout:
    sources[q - 1] = ('field', G) gives G 1_S in the mesh precision (indicator=False), ('cross', G, D, scale) the
    float64 scale G conj(D) 1_S (indicator=True: it shares the float64 store of J).
    Returns the (nrow,) float64 device sums of this rank's x slab and the number of c2r transforms run."""
    assert not (len(ells) and len(sources))
    pm = c.pm if not indicator else c.pm.reshape(dtype='f8')
    nshell = len(kedges) - 1
    nfam = len(sources) if len(sources) else len(ells)
    nfield = nshell * (1 + nfam)
    ntri = len(triples)
    dev = c.value.device
    code = _CODE[pm.typestr]
    tdt = torch.float64 if pm.typestr == 'f8' else torch.float32
    cdt = torch.complex128 if pm.typestr == 'f8' else torch.complex64
    ncell = int(numpy.prod(pm.real_shape))
    cslab = int(numpy.prod(pm.complex_shape))
    fill_n = min(_FILL_CHUNK, nfield)
    # the fill scratch, the transform's work buffers and a margin stay free
    reserve = (fill_n + 4) * cslab * torch.empty((), dtype=cdt).element_size() + (256 << 20)
    cap = _resident_cap(nfield, ncell * torch.empty((), dtype=tdt).element_size(), reserve, pm.comm)
    # row groups, each run with its fields resident: everything at once; or one family at a time (its rows need
    # W of that family and I); or, per family, shell blocks of cap // 3 so that any three of them are resident
    # together.  A row's family is that of its first field (b and c are I fields).
    rfam = triples[:, 0] // nshell
    if cap >= nfield:
        bsz, rfam = nshell, numpy.zeros_like(rfam)
    else:
        bsz = nshell if cap >= 2 * nshell else cap // 3
    key = numpy.column_stack([rfam, (triples % nshell) // bsz])   # (nrow, 4); shell blocks non-decreasing in b, c
    order = (numpy.lexsort((key[:, 3], key[:, 2], key[:, 1], key[:, 0])) if ntri
             else numpy.zeros(0, dtype='i8'))
    store = torch.empty((min(cap, nfield), ncell), dtype=tdt, device=dev)
    scratch = torch.empty((fill_n,) + tuple(pm.complex_shape), dtype=cdt, device=dev)
    out = torch.zeros(ntri, dtype=torch.float64, device=dev)
    tr, start, count = c._slab()
    k2edges = _lib.darr((numpy.asarray(kedges) ** 2).astype('f8'))
    los = _lib.darr([float(v) for v in los]) if len(ells) else None
    slot_of = {}                                          # resident field -> row of `store`
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
        # contiguous runs of missing family-0 shells, each filled in chunks of at most fill_n shells by one read of c
        runs = []
        for s in missing:
            if s >= nshell:
                break
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
        # families with their own sources: contiguous runs of missing shells, one read of the source per run
        for f, src in enumerate(sources, 1):
            fruns = []
            for s in [s % nshell for s in missing if s // nshell == f]:
                if fruns and fruns[-1][-1] == s - 1 and len(fruns[-1]) < fill_n:
                    fruns[-1].append(s)
                else:
                    fruns.append([s])
            for run in fruns:
                _fill_source(src, kedges, k2edges, run, tr, start, count, scratch, cslab)
                for q, s in enumerate(run):
                    with stage("bispec_c2r"):
                        ComplexField(pm, scratch[q]).c2r(out=RealField(pm, store[slot_of[f * nshell + s]].view(pm.real_shape)))
                    transforms += 1
        # the missing weighted fields: one read of c per chunk of families x contiguous shells
        for fams, run in _pole_chunks([s for s in missing if s >= nshell] if len(ells) else [], nshell, fill_n):
            with stage("bispec_fill_poles"):
                check(lib().nbk_bispec_fill_poles(_ptr(c.value), code, pm._nmesh_c, pm._box_c, tr, start, count, k2edges,
                                                  len(kedges), run[0], len(run), los,
                                                  _lib.i32arr([ells[f - 1] for f in fams]), len(fams), _ptr(scratch),
                                                  cslab, _stream()), "nbk_bispec_fill_poles")
            for q, f in enumerate(fams):
                for p, s in enumerate(run):
                    with stage("bispec_c2r"):
                        ComplexField(pm, scratch[q * len(run) + p]).c2r(
                            out=RealField(pm, store[slot_of[f * nshell + s]].view(pm.real_shape)))
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


def _fill_source(src, kedges, k2edges, run, tr, start, count, scratch, cslab):
    """one read of a shell_pass source field writes its shells `run` (contiguous) into the scratch slabs"""
    G = src[1]
    pm = G.pm
    if src[0] == 'field':
        with stage("bispec_fill"):
            check(lib().nbk_bispec_fill(_ptr(G.value), _CODE[pm.typestr], pm._nmesh_c, pm._box_c, tr, start, count, k2edges,
                                        len(kedges), run[0], len(run), 0, _ptr(scratch), cslab, _stream()), "nbk_bispec_fill")
    else:
        D, scale = src[2], float(src[3])
        with stage("bispec_fill_cross"):
            check(lib().nbk_bispec_fill_cross(_ptr(G.value), _ptr(D.value), _CODE[pm.typestr], pm._nmesh_c, pm._box_c, tr,
                                              start, count, k2edges, len(kedges), run[0], len(run), scale, _ptr(scratch),
                                              cslab, _stream()), "nbk_bispec_fill_cross")


def _pole_chunks(fields, nshell, fill_n):
    """(families, shells) chunks of the weighted field ids `fields` (family * nshell + shell, family >= 1), each filled
    by one nbk_bispec_fill_poles call into at most fill_n scratch slabs: contiguous shells that miss the same set of
    families, len(families) * len(shells) <= fill_n"""
    fams_of = {}
    for fid in sorted(fields):
        fams_of.setdefault(fid % nshell, []).append(fid // nshell)
    chunks = []
    for s in sorted(fams_of):
        fams = fams_of[s]
        if len(fams) > fill_n:
            chunks += [(fams[i:i + fill_n], [s]) for i in range(0, len(fams), fill_n)]
        elif (chunks and chunks[-1][0] == fams and chunks[-1][1][-1] == s - 1
              and len(fams) * (len(chunks[-1][1]) + 1) <= fill_n):
            chunks[-1][1].append(s)
        else:
            chunks.append((fams, [s]))
    return chunks


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
