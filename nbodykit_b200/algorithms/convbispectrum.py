"""
ConvolvedFFTBispectrum -- bispectrum multipoles of a survey catalogue from the FKP field with the end-point line of sight
(Scoccimarro 2015, arXiv:1506.02729 §IV; DESIGN.md 4.15).  The reference has no bispectrum: this extends the package
past it, with ConvolvedFFTPower's conventions for the field, the window compensation, alpha and the normalisation.

F is FKPCatalogMesh.to_real_field() (mass u = w_c w_fkp Value per object), c = r2c(F), compensated.  G_0 = c and, for
even ell > 0, G_ell = 4 pi sum_m Y_lm(qhat) r2c[F Y_lm(xhat)] = (2 ell + 1) r2c[F L_ell(qhat.xhat)], compensated
(ConvolvedFFTPower's A_ell, fkp.ylm_multipole).  Per k shell S_a: I_a = c2r(c 1_Sa), W^ell_a = c2r(G_ell 1_Sa) (mesh
precision), J_a = c2r(1_Sa) (float64); for every row (a, b, c), b <= c, of an evaluated triple

    B_ell[a, b, c] = V^3 sum_x W^ell_a I_b I_c / (I33 sum_x J_a J_b J_c),    W^0 = I,  I33 = randoms.norm3

Shot noise of the monopole, exact (the coincident-object terms of the raw estimator): N is painted as F with mass u^2
and +alpha^2 for the randoms, c_N = r2c(N) compensated, H_a = c2r(V^2 c conj(c_N) 1_Sa) (float64), S3 = sum_d u^3 -
alpha^3 sum_r u^3 and

    shotnoise_0[a, b, c] = [sum_x (H_a J_b J_c + J_a H_b J_c + J_a J_b H_c) / sum_x J_a J_b J_c - 2 S3] / I33

It is NOT subtracted.  The fills, the shell transforms and the triple sums are bispectrum.shell_pass's.
"""
import logging

import numpy
import torch

from .. import CurrentMPIComm
from .._lib import stage
from ..binned_statistic import BinnedStatistic
from ..pmesh.pm import ComplexField, RealField
from ..utils import JSONDecoder, JSONEncoder
from .bispectrum import bispectrum_table, pole_triples, shell_edges, shell_pass, shell_triples, _MAX_ELL
from .convpower.fkp import _cast_mesh, copy_meta, get_compensation, ylm_multipole
from .fftpower import project_to_basis_device


def check_convolved_poles(poles):
    """the validated multipole list (ints): even ell, 0 <= ell <= 8 (the Y_lm table limit), no repeat; raises ValueError
    before any device work.  Odd ell are imaginary with an end-point line of sight."""
    poles = [poles] if numpy.isscalar(poles) else list(poles)
    if not poles:
        raise ValueError("ConvolvedFFTBispectrum: poles is empty")
    for ell in poles:
        if numpy.ndim(ell) != 0 or int(ell) != ell or not 0 <= ell <= _MAX_ELL:
            raise ValueError("ConvolvedFFTBispectrum: multipole %r; poles must be even integers 0 <= ell <= %d (the "
                             "Y_lm table limit)" % (ell, _MAX_ELL))
        if ell % 2:
            raise ValueError("ConvolvedFFTBispectrum: odd multipole ell = %d; with an end-point line of sight an odd ell "
                             "gives an imaginary statistic" % ell)
    if len(set(poles)) != len(poles):
        raise ValueError("ConvolvedFFTBispectrum: repeated multipole in poles = %r" % (poles,))
    return [int(ell) for ell in poles]


def convolved_table(kedges, kmean, triples, prows, S, W, Tsum, Hsum, volume, I33, S3, Ncells, poles):
    """the (n, n, n) structured array of `.poles`: k1, k2, k3, B_<ell> per requested ell, shotnoise_0 (0 in poles),
    triangles.  S = sum_x I I I and Tsum = sum_x J J J per sorted triple of `triples`; W[ell] = sum_x G-weighted
    W^ell_a I_b I_c per row (a, b, c) of `prows` (pole_triples), already multiplied by 4 pi; Hsum = sum_x H_a J_b J_c per
    row of `prows` (or None).  Entries whose sorted triple is not evaluated or holds no triangle report NaN."""
    base = bispectrum_table(kedges, kmean, triples, numpy.asarray(S, dtype='f8') * (volume / I33), Tsum, volume, Ncells)
    n = len(kedges) - 1
    fields = [('k1', 'f8'), ('k2', 'f8'), ('k3', 'f8')] + [('B_%d' % ell, 'f8') for ell in poles]
    if 0 in poles:
        fields.append(('shotnoise_0', 'f8'))
    data = numpy.zeros((n, n, n), dtype=fields + [('triangles', 'i8')])
    for f in ('k1', 'k2', 'k3', 'triangles'):
        data[f] = base[f]
    if 0 in poles:
        data['B_0'] = base['B']
    triples = numpy.asarray(triples).reshape(-1, 3)
    prows = numpy.asarray(prows).reshape(-1, 3)
    index = {tuple(t): q for q, t in enumerate(triples.tolist())}
    tri = numpy.array([index[tuple(sorted(r))] for r in prows.tolist()], dtype='i8')
    Tsum = numpy.asarray(Tsum, dtype='f8')
    count = base['triangles'][triples[:, 0], triples[:, 1], triples[:, 2]]
    rcount = count[tri] if len(prows) else numpy.zeros(0, dtype='i8')
    for ell in poles:
        if ell == 0:
            continue
        with numpy.errstate(invalid='ignore', divide='ignore'):
            B = numpy.where(rcount > 0, volume ** 3 * numpy.asarray(W[ell], dtype='f8') / (I33 * Tsum[tri]), numpy.nan)
        col = numpy.full((n, n, n), numpy.nan)
        col[prows[:, 0], prows[:, 1], prows[:, 2]] = B
        col[prows[:, 0], prows[:, 2], prows[:, 1]] = B
        data['B_%d' % ell] = col
    if 0 in poles:
        # sum_x (H_a J_b J_c + J_a H_b J_c + J_a J_b H_c) of a sorted triple: each distinct shell a once per occurrence
        mult = numpy.array([list(triples[t]).count(r[0]) for t, r in zip(tri, prows.tolist())], dtype='f8')
        hs = numpy.zeros(len(triples))
        numpy.add.at(hs, tri, mult * numpy.asarray(Hsum, dtype='f8'))
        with numpy.errstate(invalid='ignore', divide='ignore'):
            sn = numpy.where(count > 0, (hs / Tsum - 2 * S3) / I33, numpy.nan)
        col = numpy.full((n, n, n), numpy.nan)
        for (i, j, l), v in zip(triples.tolist(), sn):
            for p in {(i, j, l), (i, l, j), (j, i, l), (j, l, i), (l, i, j), (l, j, i)}:
                col[p] = v
        data['shotnoise_0'] = col
    return data


class ConvolvedFFTBispectrum(object):
    """
    Bispectrum multipoles of a survey catalogue about the end-point line of sight (Scoccimarro 2015 §IV), from the FKP
    field of ConvolvedFFTPower.

    first : FKPCatalog or FKPCatalogMesh     cast as ConvolvedFFTPower casts it; 'f4', 'f8', 'c8', 'c16' meshes
    poles : list of int                      even ell, 0 <= ell <= 8
    Nmesh, dk, kmin, kmax                    the shells of FFTBispectrum (bispectrum.shell_edges)

    For every evaluated shell row (a, b, c), b <= c (the Legendre weight on k1, shell a):

        B_ell[a, b, c] = V^3 sum_x W^ell_a I_b I_c / (I33 sum_x J_a J_b J_c)

    with W^ell_a = c2r(G_ell 1_Sa), G_ell = (2 ell + 1) r2c[F L_ell(qhat.xhat)], I = W^0 and I33 = ``randoms.norm3`` =
    alpha sum_r nbar^2 w_c w_fkp^3 (1 without randoms).  B_0 is symmetric in all three indices, B_ell in (b, c) only.
    For a periodic field F = nbar (1 + delta) with unit weights I33 = nbar^3 V and B_0 is FFTBispectrum's B.
    ``shotnoise_0`` is the exact monopole shot noise (the coincident-object terms); it is NOT subtracted, and B_ell > 0
    is reported raw.

    Results, computed in __init__: ``.poles`` (BinnedStatistic, dims k1, k2, k3; fields k1, k2, k3 -- the shells' mean
    |k| --, B_<ell>, shotnoise_0 when 0 is in poles, triangles), ``.edges`` and ``.attrs`` (``transforms`` counts the
    r2c and c2r transforms run).  When the shell fields do not fit in device memory (or NBK_BISPEC_RESIDENT caps them)
    they are built per block of shells, as in FFTBispectrum.
    """
    logger = logging.getLogger('ConvolvedFFTBispectrum')

    def __init__(self, first, poles=[0], Nmesh=None, dk=None, kmin=0., kmax=None):
        poles = check_convolved_poles(poles)
        first = _cast_mesh(first, Nmesh=Nmesh)
        self.first = first
        self.comm = first.comm
        self.attrs = {}
        self.attrs['poles'] = poles
        if dk is None:
            dk = 2 * numpy.pi / numpy.min(first.attrs['BoxSize'])
        self.attrs['dk'] = dk
        self.attrs['kmin'] = kmin
        self.attrs['kmax'] = kmax
        self.attrs['Nmesh'] = first.attrs['Nmesh'].copy()
        self.attrs['BoxSize'] = first.attrs['BoxSize']
        self.attrs['BoxPad'] = first.attrs['BoxPad']
        self.attrs['BoxCenter'] = first.attrs['BoxCenter']
        self.attrs['mesh.resampler'] = first.resampler
        self.attrs['mesh.interlaced'] = first.interlaced
        # the shells are validated (dk = 0, kmin < 0, no shell, too many) before any paint or transform
        self.edges = shell_edges(self.attrs['Nmesh'], self.attrs['BoxSize'], dk, kmin, kmax)
        self.run()

    def run(self):
        mesh = self.first
        kedges = self.edges
        poles = self.attrs['poles']
        ells = sorted(ell for ell in poles if ell > 0)
        nshell = len(kedges) - 1
        triples = shell_triples(kedges)
        prows = pole_triples(kedges)
        rank = self.comm.rank

        # the compensation is applied to every complex field here, not by the mesh actions
        mesh._actions[:] = []
        comp = get_compensation(mesh)
        mesh.compensated = False
        with stage("H:paint"):
            rfield = mesh.compute(mode='real')
        meta = rfield.attrs.copy()
        alpha = meta['alpha']
        self.attrs['alpha'] = alpha
        pm = rfield.pm
        V = float(numpy.prod(pm.BoxSize))
        with stage("convbispec_r2c"):
            c = rfield.r2c()
            if comp is not None:
                c.compensate(comp)
        transforms = 1
        G = {}
        if ells:
            offset = self.attrs['BoxCenter'] + 0.5 * pm.BoxSize / pm.Nmesh
            work_r, work_c = RealField(pm), ComplexField(pm)
            for ell in ells:
                with stage("convbispec_ylm"):
                    G[ell] = ylm_multipole(rfield, ell, offset, ComplexField(pm), work_r, work_c)
                    if comp is not None:
                        G[ell].compensate(comp)
                transforms += 2 * ell + 1
            del work_r, work_c
        del rfield

        for name in ('data', 'randoms'):
            self.attrs[name + '.norm3'] = self._norm3(name, alpha)
        Adata, Aran = self.attrs['data.norm3'], self.attrs['randoms.norm3']
        if Aran > 0:
            if not numpy.allclose(Adata, Aran, rtol=0.05):
                raise ValueError("normalization in ConvolvedFFTBispectrum different by more than 5%%; algorithm requires "
                                 "they must be similar\n\trandoms.norm3 = %.6f, data.norm3 = %.6f\n\tn(z) columns for "
                                 "'data' and 'randoms' should be normalized to represent n(z) of the data catalog"
                                 % (Aran, Adata))
            I33 = Aran
        else:
            I33 = 1.0
            if rank == 0:
                self.logger.info("normalization of the bispectrum is neglected, as no random is provided.")
        self.attrs['S3'] = self._s3(alpha)

        # the shells' mean |k| through FFTPower's binning, k = 0 left out as FFTBispectrum leaves it out
        result, _ = project_to_basis_device(c, [kedges, numpy.array([-1., 1.])], is_p3d=False, volume=V, need_mu=False)
        xmean, _, _, modes = [numpy.asarray(r)[:, 0] for r in result]
        kmean = xmean.copy()
        if kedges[0] == 0 and modes[0] > 1:
            kmean[0] = xmean[0] * modes[0] / (modes[0] - 1)

        # I pass: the sorted triples over I, then per ell > 0 the rows (W^ell_a, I_b, I_c)
        rows = numpy.concatenate([triples] + [prows + numpy.array([(q + 1) * nshell, 0, 0], dtype='i4')
                                              for q in range(len(ells))])
        sI, n = shell_pass(c, kedges, rows, False, sources=[('field', G[ell]) for ell in ells])
        transforms += n
        del G
        # J pass: the sorted triples over J, then (0 in poles) the rows (H_a, J_b, J_c) of the shot noise
        jsources, jrows = [], triples
        if 0 in poles:
            with stage("H:paint_shot"):
                nfield = mesh.to_shot_field()
            with stage("convbispec_r2c"):
                cN = nfield.r2c()
                if comp is not None:
                    cN.compensate(comp)
            del nfield
            transforms += 1
            jsources = [('cross', c, cN, V * V)]
            jrows = numpy.concatenate([triples, prows + numpy.array([nshell, 0, 0], dtype='i4')])
        sJ, n = shell_pass(c, kedges, jrows, True, sources=jsources)
        transforms += n
        packed = torch.cat([sI, sJ])
        with stage("bispec_allreduce"):
            if pm.comm.size > 1:
                pm.comm.allreduce_tensor(packed)
        host = packed.cpu().numpy()
        ntri, nrow, npr = len(triples), len(rows), len(prows)
        W = {ell: 4 * numpy.pi * host[ntri + q * npr:ntri + (q + 1) * npr] for q, ell in enumerate(ells)}
        Tsum = host[nrow:nrow + ntri]
        Hsum = host[nrow + ntri:] if 0 in poles else None
        data = convolved_table(kedges, kmean, triples, prows, host[:ntri], W, Tsum, Hsum, V, I33, self.attrs['S3'],
                               int(numpy.prod(pm.Nmesh)), poles)
        self.attrs['transforms'] = transforms
        copy_meta(self.attrs, meta)
        self.poles = BinnedStatistic(['k1', 'k2', 'k3'], [kedges] * 3, data, **self.attrs)
        return self.poles

    def _species_sum(self, name, f):
        """sum over the selected objects of species `name` of the column expression f(nbar, w_c, w_fkp, Value)
        (allreduced)"""
        from ..base.catalog import ConstantColumn
        mesh = self.first
        cat = mesh.source[name]
        x = f(cat[mesh.nbar], cat[mesh.comp_weight], cat[mesh.fkp_weight], cat[mesh.value])
        sel = cat[mesh.selection]
        if not (isinstance(sel, ConstantColumn) and bool(sel.value)):
            x = x[sel]
        return self.comm.allreduce(float(x.sum()))

    def _norm3(self, name, alpha):
        """sum nbar^2 w_c w_fkp^3 over the selected objects, times alpha for the randoms"""
        A = self._species_sum(name, lambda nbar, wc, wf, v: nbar ** 2 * wc * wf ** 3)
        return A * alpha if name == 'randoms' else A

    def _s3(self, alpha):
        """S3 = sum_d u^3 - alpha^3 sum_r u^3, u = w_c w_fkp Value"""
        u3 = lambda nbar, wc, wf, v: (wc * wf * v) ** 3          # noqa: E731
        return self._species_sum('data', u3) - alpha ** 3 * self._species_sum('randoms', u3)

    def __getstate__(self):
        return dict(poles=self.poles.__getstate__(), attrs=self.attrs, edges=self.edges)

    def __setstate__(self, state):
        self.attrs = state['attrs']
        self.edges = numpy.asarray(state['edges'])
        self.poles = BinnedStatistic.from_state(state['poles'])

    def save(self, output):
        import json
        if self.comm.rank == 0:
            self.logger.info('saving ConvolvedFFTBispectrum result to %s' % output)
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

