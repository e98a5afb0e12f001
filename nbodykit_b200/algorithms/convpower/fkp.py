"""
ConvolvedFFTPower -- window-convolved power spectrum multipoles of a survey catalogue
(API of nbodykit/algorithms/convpower/fkp.py:76-797; estimator of Hand et al. 2017: 2l+1 FFTs per l).

Where the O(Nmesh^3) work runs (reference line numbers):
  F(x)               FKPCatalogMesh.to_real_field: two paints, one axpy, one scale          (catalogmesh.py:122-204)
  A_0 = V FFT[F]     one r2c; the factor V and the window compensation are folded into the binning kernel (:478-487)
  A_l = 4 pi V sum_m Y_lm(khat) FFT[F Y_lm(xhat)]    per m: nbk_ylm_mul_real -> r2c -> nbk_ylm_mul_complex_acc
                     (the reference builds six full-size f8 unit-vector arrays :531-538; here xhat / khat are
                     formed on the fly)                                                     (:571-597)
  P_l = <norm A_0 A_l^*>_k   nbk_power_bin(c1 = FFT[F], c2 = sum_m ..., volume = norm 4 pi V^2, comp1, comp2),
                     zero mode NOT cleared, mu edges (-1, 1)                                (:605-623, 631-643)
Meshes are stored Hermitian-compressed; the reference's default 'c16' complex mesh is accepted and reproduced through
the anti-Hermitian fold of the odd multipoles (no c2c transform is needed: the FKP field is real in configuration space).
"""
import logging
import time
import warnings

import numpy

from ... import CurrentMPIComm, _lib
from ..._lib import check, lib
from ...binned_statistic import BinnedStatistic
from ...pmesh.pm import ComplexField, RealField, _CODE, _ptr, _stream
from ...utils import JSONDecoder, JSONEncoder, timer
from ..fftpower import _find_unique_edges, project_to_basis_device
from .catalog import FKPCatalog
from .catalogmesh import FKPCatalogMesh

# largest l of the real spherical harmonics the device evaluates (NBK_YLM_LMAX of csrc/ylm_table.inc, tools/gen_ylm.py)
YLM_LMAX = 8


class ConvolvedFFTPower(object):
    """
    first : FKPCatalog or FKPCatalogMesh
    poles : list of int            multipoles to compute
    second : FKPCatalog(Mesh), optional     cross-correlation (same data/randoms, different weights)
    Nmesh, kmin, kmax, dk : binning (dk=None -> 2 pi / min(BoxSize); dk=0 -> one bin per unique |k|)

    Results: `.poles` (BinnedStatistic over 'k': `k`, `power_L` (complex64), `modes`), `.edges`, `.attrs`
    (`alpha`, `data.norm`, `randoms.norm`, `shotnoise`, per-species N/W/W2/num_per_cell, box geometry).
    """
    logger = logging.getLogger('ConvolvedFFTPower')

    def __init__(self, first, poles, second=None, Nmesh=None, kmin=0., kmax=None, dk=None, use_fkp_weights=None,
                 P0_FKP=None):
        if use_fkp_weights is not None or P0_FKP is not None:
            raise ValueError("use_fkp_weights and P0_FKP are deprecated. Assign a FKPWeight column to "
                             "source['randoms']['FKPWeight'] and source['data']['FKPWeight'] with the help of "
                             "the FKPWeightFromNbar(nbar) function")
        # Y_lm exists on the device up to the generated table's l (csrc/ylm_table.inc): refuse larger l before any
        # paint or FFT runs
        if any(int(ell) > YLM_LMAX for ell in numpy.atleast_1d(poles)):
            raise ValueError("ConvolvedFFTPower computes multipoles l <= %d (the Y_lm table limit); got poles=%s"
                             % (YLM_LMAX, list(numpy.atleast_1d(poles))))
        first = _cast_mesh(first, Nmesh=Nmesh)
        if second is not None:
            second = _cast_mesh(second, Nmesh=Nmesh)
        else:
            second = first
        if not is_valid_crosscorr(first, second):
            raise NotImplementedError("ConvolvedFFTPower cross-correlations currently require the same"
                                      " FKPCatalog (data/randoms), such that only the weight column can vary")
        self.first = first
        self.second = second
        self.comm = first.comm
        if not numpy.array_equal(first.attrs['BoxSize'], second.attrs['BoxSize']):
            joint = {}
            for name in ['BoxSize', 'BoxCenter']:
                joint[name] = numpy.vstack([first.attrs[name], second.attrs[name]])
            argmax = numpy.argmax(joint['BoxSize'], axis=0)
            joint['BoxSize'] = joint['BoxSize'][argmax, [0, 1, 2]]
            joint['BoxCenter'] = joint['BoxCenter'][argmax, [0, 1, 2]]
            first.recenter_box(joint['BoxSize'], joint['BoxCenter'])
            second.recenter_box(joint['BoxSize'], joint['BoxCenter'])
        if numpy.isscalar(poles):
            poles = [poles]
        self.attrs = {}
        self.attrs['poles'] = poles
        self.attrs['dk'] = dk
        self.attrs['kmin'] = kmin
        self.attrs['kmax'] = kmax
        self.attrs['Nmesh'] = self.first.attrs['Nmesh'].copy()
        self.attrs['BoxSize'] = self.first.attrs['BoxSize']
        self.attrs['BoxPad'] = self.first.attrs['BoxPad']
        self.attrs['BoxCenter'] = self.first.attrs['BoxCenter']
        self.attrs['mesh.resampler'] = self.first.resampler
        self.attrs['mesh.interlaced'] = self.first.interlaced
        self.run()

    def run(self):
        pm = self.first.pm
        dk = 2 * numpy.pi / pm.BoxSize.min() if self.attrs['dk'] is None else self.attrs['dk']
        kmin = self.attrs['kmin']
        kmax = self.attrs['kmax']
        if kmax is None:
            kmax = numpy.pi * pm.Nmesh.min() / pm.BoxSize.max() + dk / 2
        if dk > 0:
            kedges = numpy.arange(kmin, kmax, dk)
            kcoords = None
        else:
            kedges, kcoords = _find_unique_edges(pm, kmax)
            if self.comm.rank == 0:
                self.logger.info('%d unique k values are found' % len(kcoords))
        result = self._compute_multipoles(kedges)
        self.poles = BinnedStatistic(['k'], [kedges], result, fields_to_sum=['modes'], coords=[kcoords], **self.attrs)
        self.edges = kedges

    def to_pkmu(self, mu_edges, max_ell):
        """invert the multipoles into wedges P(k, mu) = sum_l P_l(k) <L_l(mu)>_bin  (fkp.py:282-338)"""
        from scipy.special import legendre
        from scipy.integrate import quad

        def coefficient(ell, mumin, mumax):
            return quad(lambda mu: legendre(ell)(mu), mumin, mumax)[0] / (mumax - mumin)
        ells = list(range(0, max_ell + 1, 2))
        if any('power_%d' % ell not in self.poles for ell in ells):
            raise ValueError("measurements for ells=%s required if max_ell=%d" % (ells, max_ell))
        dtype = numpy.dtype([('power', 'c8'), ('k', 'f8'), ('mu', 'f8')])
        data = numpy.zeros((self.poles.shape[0], len(mu_edges) - 1), dtype=dtype)
        for imu, (lo, hi) in enumerate(zip(mu_edges[:-1], mu_edges[1:])):
            for ell in ells:
                data['power'][:, imu] += coefficient(ell, lo, hi) * self.poles['power_%d' % ell]
            data['k'][:, imu] = self.poles['k']
            data['mu'][:, imu] = numpy.ones(len(data)) * 0.5 * (hi + lo)
        return BinnedStatistic(dims=['k', 'mu'], edges=[self.poles.edges['k'], mu_edges], data=data,
                               coords=[self.poles.coords['k'], None], **self.attrs)

    def __getstate__(self):
        return dict(poles=self.poles.__getstate__(), attrs=self.attrs)

    def __setstate__(self, state):
        self.attrs = state['attrs']
        self.poles = BinnedStatistic.from_state(state['poles'])

    def save(self, output):
        import json
        if self.comm.rank == 0:
            self.logger.info('saving ConvolvedFFTPower result to %s' % output)
            with open(output, 'w') as ff:
                json.dump(self.__getstate__(), ff, cls=JSONEncoder)

    @classmethod
    @CurrentMPIComm.enable
    def load(cls, output, comm=None, format='current'):
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

    # ------------------------------------------------------------------------------------------------
    def _compute_multipoles(self, kedges):
        # the compensation is applied here (fused into the binning), not by the mesh actions
        for source in [self.first, self.second]:
            source._actions[:] = []
        compensation = {}
        for name, mesh in zip(['first', 'second'], [self.first, self.second]):
            compensation[name] = get_compensation(mesh)
            mesh.compensated = False
            if self.comm.rank == 0:
                if compensation[name] is not None:
                    self.logger.info("using compensation function %s for source '%s'" % (compensation[name], name))
                else:
                    self.logger.warning("no compensation applied for source '%s'" % name)
        rank = self.comm.rank
        pm = self.first.pm
        muedges = numpy.linspace(-1, 1, 2, endpoint=True)
        edges = [kedges, muedges]
        cols = ['k'] + ['power_%d' % l for l in sorted(self.attrs['poles'])] + ['modes']
        dtype = ['f8'] + ['c8'] * len(self.attrs['poles']) + ['i8']
        result = numpy.empty(len(kedges) - 1, dtype=numpy.dtype(list(zip(cols, dtype))))
        offset = self.attrs['BoxCenter'] + 0.5 * pm.BoxSize / pm.Nmesh
        poles = sorted(self.attrs['poles'])
        if 0 not in poles:
            poles = [0] + poles
        assert poles[0] == 0

        rfield1 = self.first.compute(mode='real')
        meta1 = rfield1.attrs.copy()
        if rank == 0:
            self.logger.info("%s painting of 'first' done" % self.first.resampler)
        self.attrs['alpha'] = meta1['alpha']
        c1 = rfield1.r2c()
        if rank == 0:
            self.logger.info('ell = 0 done; 1 r2c completed')
        volume = float(pm.BoxSize.prod())

        c2_0 = None
        if self.first is not self.second:
            rfield2 = self.second.compute(mode='real')
            meta2 = rfield2.attrs.copy()
            if rank == 0:
                self.logger.info("%s painting of 'second' done" % self.second.resampler)
            if 0 in self.attrs['poles']:
                c2_0 = rfield2.r2c()
        else:
            rfield2 = rfield1
            meta2 = meta1
            if 0 in self.attrs['poles']:
                c2_0 = c1
        if not numpy.allclose(rfield1.attrs['alpha'], rfield2.attrs['alpha'], rtol=1e-3):
            raise ValueError("ConvolvedFFTPower cross-correlations currently require the same"
                             " FKPCatalog (data/randoms), such that only the weight column can vary;"
                             " different ``alpha`` values found for first/second meshes")

        for name in ['data', 'randoms']:
            self.attrs[name + '.norm'] = self.normalization(name, self.attrs['alpha'])
        if self.attrs['randoms.norm'] > 0:
            norm = 1.0 / self.attrs['randoms.norm']
            Adata, Aran = self.attrs['data.norm'], self.attrs['randoms.norm']
            if not numpy.allclose(Adata, Aran, rtol=0.05):
                msg = "normalization in ConvolvedFFTPower different by more than 5%; "
                msg += ",algorithm requires they must be similar\n"
                msg += "\trandoms.norm = %.6f, data.norm = %.6f\n" % (Aran, Adata)
                msg += "\tpossible discrepancies could be related to normalization "
                msg += "of n(z) column ('%s')\n" % self.first.nbar
                msg += "\tor the consistency of the FKP weight column for 'data' and 'randoms';\n"
                msg += "\tn(z) columns for 'data' and 'randoms' should be normalized to represent n(z) of the data catalog"
                raise ValueError(msg)
            if rank == 0:
                self.logger.info("normalized power spectrum with `randoms.norm = %.6f`" % Aran)
        else:
            norm = 1.0
            if rank == 0:
                self.logger.info("normalization of power spectrum is neglected, as no random is provided.")

        comp = (compensation['first'], compensation['second'])
        code = _CODE[pm.typestr]
        tr, cstart, ccount = c1._slab()
        off_c = _lib.darr(offset)
        proj = None
        start = time.time()
        # complex ('c16' / 'c8') meshes: the reference sums over ALL modes of a full mesh.  The field is real in
        # configuration space, so the unstored half follows from the stored one -- except that Y_lm(khat) at the mirror
        # of a mode with a Nyquist component is not (-1)^l Y_lm(khat) (the Nyquist label stays -N/2): Bell accumulates
        # the A_l the mirror modes carry, and the binning kernel takes the mirror half from it (nbk_power_bin2)
        full_mesh = bool(getattr(self.first, 'complex_mesh', False))
        if len(poles) > 1:
            Aell = ComplexField(pm)
            Bell = ComplexField(pm) if full_mesh else None
            work_r = RealField(pm)
            work_c = ComplexField(pm)
        for ell in poles[1:]:
            Aell[...] = 0.
            if full_mesh:
                Bell[...] = 0.
            substart = time.time()
            for m in range(-ell, ell + 1):
                # F(x) Y_lm(xhat) -> FFT -> accumulate Y_lm(khat) * FFT
                check(lib().nbk_ylm_mul_real(_ptr(rfield2.value), _ptr(work_r.value), code, ell, m, pm._nmesh_c,
                                             pm._box_c, off_c, pm.x_start, pm.x_n, _stream()), "nbk_ylm_mul_real")
                work_r.r2c(out=work_c)
                if full_mesh:
                    check(lib().nbk_ylm_mul_complex_acc2(_ptr(Aell.value), _ptr(Bell.value), _ptr(work_c.value), code, ell, m,
                                                         pm._nmesh_c, pm._box_c, tr, cstart, ccount, _stream()),
                          "nbk_ylm_mul_complex_acc2")
                else:
                    check(lib().nbk_ylm_mul_complex_acc(_ptr(Aell.value), _ptr(work_c.value), code, ell, m, pm._nmesh_c,
                                                        pm._box_c, tr, cstart, ccount, _stream()), "nbk_ylm_mul_complex_acc")
                if rank == 0:
                    self.logger.debug("done term for Y(l=%d, m=%d) in %s" % (ell, m, timer(substart, time.time())))
            if rank == 0:
                self.logger.info('ell = %d done; %s r2c completed' % (ell, 2 * ell + 1))
            # P_l = < norm * (V c1 / comp1) * conj(4 pi V Aell / comp2) >
            # complex meshes: the true sum over all N^3 modes (mirror half from Bell); Hermitian ('f8'/'f4') meshes keep
            # the reference's own Hermitian fold (documented there as incorrect for odd ell)
            proj, _ = project_to_basis_device(c1, edges, second=Aell, is_p3d=False,
                                              volume=norm * 4 * numpy.pi * volume * volume, compensation=comp,
                                              clear_zero=False, mirror=Bell if full_mesh else None)
            result['power_%d' % ell][:] = numpy.squeeze(proj[2])
        if rank == 0:
            self.logger.info("higher order multipoles computed in elapsed time %s" % timer(start, time.time()))
        if 0 in self.attrs['poles'] or proj is None:
            proj, _ = project_to_basis_device(c1, edges, second=c2_0 if c2_0 is not c1 else None, is_p3d=False,
                                              volume=norm * volume * volume, compensation=comp, clear_zero=False)
            if 0 in self.attrs['poles']:
                result['power_0'][:] = numpy.squeeze(proj[2])
        result['k'][:] = numpy.squeeze(proj[0])
        result['modes'][:] = numpy.squeeze(proj[-1])
        self.attrs['shotnoise'] = self.shotnoise(self.attrs['alpha'])
        if self.first is self.second:
            copy_meta(self.attrs, meta1)
        else:
            copy_meta(self.attrs, meta1, prefix='first')
            copy_meta(self.attrs, meta2, prefix='second')
        return result

    def _selected(self, mesh, name):
        cat = mesh.source[name]
        from ...base.catalog import ConstantColumn
        sel = cat[mesh.selection]
        if isinstance(sel, ConstantColumn) and bool(sel.value):
            return cat, None
        return cat, sel

    def normalization(self, name, alpha):
        """A = sum nbar w_comp w_fkp1 w_fkp2 (x alpha for the randoms)   (fkp.py:657-709)"""
        assert name in ['data', 'randoms']
        if name + '.norm' not in self.attrs:
            first, sel = self._selected(self.first, name)
            second, _ = self._selected(self.second, name)
            comp_weight = first[self.first.comp_weight]
            nbar = second[self.second.nbar]
            fkp1 = first[self.first.fkp_weight]
            fkp2 = fkp1 if self.first is self.second else second[self.second.fkp_weight]
            A = nbar * comp_weight * fkp1 * fkp2
            if sel is not None:
                A = A[sel]
            A = float(A.sum())
            if name == 'randoms':
                A *= alpha
            self.attrs[name + '.norm'] = self.comm.allreduce(A)
        return self.attrs[name + '.norm']

    def shotnoise(self, alpha):
        """S = [sum_d (w_c^2 w_fkp1 w_fkp2) + alpha^2 sum_r (...)] / randoms.norm   (fkp.py:711-759)"""
        if 'shotnoise' not in self.attrs:
            Pshot = 0
            for name in ['data', 'randoms']:
                first, sel = self._selected(self.first, name)
                second, _ = self._selected(self.second, name)
                comp_weight = first[self.first.comp_weight]
                fkp1 = first[self.first.fkp_weight]
                fkp2 = fkp1 if self.first is self.second else second[self.second.fkp_weight]
                S = comp_weight ** 2 * fkp1 * fkp2
                if sel is not None:
                    S = S[sel]
                S = float(S.sum())
                if name == 'randoms':
                    S *= alpha ** 2
                Pshot += S
            Pshot = self.comm.allreduce(Pshot)
            self.attrs['shotnoise'] = Pshot / self.attrs['randoms.norm'] if self.attrs['randoms.norm'] > 0 else 0.
        return self.attrs['shotnoise']


FKPPower = ConvolvedFFTPower


def _cast_mesh(mesh, Nmesh):
    if not isinstance(mesh, (FKPCatalogMesh, FKPCatalog)):
        raise TypeError("input sources should be a FKPCatalog or FKPCatalogMesh")
    if isinstance(mesh, FKPCatalog):
        mesh = mesh.to_mesh(Nmesh=Nmesh, dtype='c16', compensated=False)      # as the reference does (fkp.py:774)
    if Nmesh is not None and any(mesh.attrs['Nmesh'] != Nmesh):
        raise ValueError(("Mismatched Nmesh between __init__ and mesh.attrs; "
                          "if trying to re-sample with a different mesh, specify "
                          "`Nmesh` as keyword of to_mesh()"))
    return mesh


def get_compensation(mesh):
    """name of the compensation transfer function defined for the mesh's window (applied whenever one is
    defined, whatever `mesh.compensated` says -- the reference does the same, fkp.py:783-790), or None"""
    try:
        return mesh._get_compensation()[0][1].__name__
    except ValueError:
        return None


def copy_meta(attrs, meta, prefix=""):
    if prefix:
        prefix += '.'
    for key in meta:
        if key.startswith('data.') or key.startswith('randoms.'):
            attrs[prefix + key] = meta[key]


def is_valid_crosscorr(first, second):
    """cross-correlations need the same FKPCatalog and the same selection / completeness / n(z) columns; only the
    FKP weight column may differ (fkp.py:799-808)"""
    if second.source is not first.source:
        return False
    same_cols = ['selection', 'comp_weight', 'nbar']
    if any(getattr(second, name) != getattr(first, name) for name in same_cols):
        return False
    return True
