"""FKPCatalogMesh -- paints F(x) = w_fkp (w_c n_data - alpha w_c n_randoms) / V_cell
(API of nbodykit/algorithms/convpower/catalogmesh.py:9-244)."""
import logging

import numpy

from ...base.catalog import ConstantColumn
from ...source.mesh.catalog import CatalogMesh
from ...source.mesh.species import MultipleSpeciesCatalogMesh
from ...utils import attrs_to_dict


class FKPCatalogMesh(MultipleSpeciesCatalogMesh):
    logger = logging.getLogger('FKPCatalogMesh')

    def __init__(self, source, BoxSize, BoxCenter, Nmesh, dtype, selection, comp_weight, fkp_weight, nbar,
                 value='Value', position='Position', interlaced=False, compensated=False, resampler='cic'):
        from .catalog import FKPCatalog
        if not isinstance(source, FKPCatalog):
            raise TypeError("the input source for FKPCatalogMesh must be a FKPCatalog")
        uncentered_position = position
        position = '_RecenteredPosition'
        weight = '_TotalWeight'
        self.attrs.update(source.attrs)
        self.recenter_box(BoxSize, BoxCenter)
        # 'c16' / 'c8' (the reference's default, convpower/catalog.py:151,169-176): the FKP field is real-valued in
        # configuration space, so its transform is stored Hermitian-compressed here as well; what the full complex mesh
        # buys the reference -- correct ODD multipoles -- is obtained by folding the mirror half with the
        # anti-Hermitian sign in the binning kernel (ConvolvedFFTPower._compute_multipoles)
        self.complex_mesh = numpy.dtype(dtype).kind == 'c'
        if self.complex_mesh:
            dtype = 'f8' if numpy.dtype(dtype).itemsize == 16 else 'f4'
        MultipleSpeciesCatalogMesh.__init__(self, source=source, BoxSize=BoxSize, Nmesh=Nmesh, dtype=dtype,
                                            weight=weight, value=value, selection=selection, position=position,
                                            interlaced=interlaced, compensated=compensated, resampler=resampler)
        self._uncentered_position = uncentered_position
        self.comp_weight = comp_weight
        self.fkp_weight = fkp_weight
        self.nbar = nbar

    def __getitem__(self, key):
        return self._species_mesh(key)

    def _species_mesh(self, key, power=1):
        """the species' CatalogMesh, each object of mass u^power (u = w_c w_fkp Value)"""
        assert key in self.source.species, "the species is not defined in the source"
        cat = self.source[key]
        assert cat.comm is self.comm
        weight, value = self.TotalWeight(key), cat[self.value]
        if power != 1:
            weight, value = weight ** power, value ** power
        return CatalogMesh(cat, BoxSize=self.attrs['BoxSize'], Nmesh=self.attrs['Nmesh'], dtype=self.dtype,
                           Weight=weight, Value=value, Selection=cat[self.selection],
                           Position=self.RecenteredPosition(key), interlaced=self.interlaced,
                           compensated=self.compensated, resampler=self.resampler)

    def to_shot_field(self):
        """N = (sum_d u^2 W(x - x_d) + alpha^2 sum_r u^2 W(x - x_r)) / V_cell, painted as to_real_field paints F (same
        window and interlacing) with mass u^2 and +alpha^2 in place of -alpha: the coincident-object field of the
        bispectrum shot noise (ConvolvedFFTBispectrum)"""
        wd, wr = self.weighted_total('data'), self.weighted_total('randoms')
        alpha = wd / wr if wr != 0 else numpy.inf
        real = self._species_mesh('data', 2).to_real_field(normalize=False)
        if self.source['randoms'].csize > 0:
            real2 = self._species_mesh('randoms', 2).to_real_field(normalize=False)
            real.axpy(real2, alpha ** 2)
            del real2
        real /= (self.pm.BoxSize / self.pm.Nmesh).prod()
        real.attrs = {'alpha': alpha}
        return real

    def recenter_box(self, BoxSize, BoxCenter):
        """positions are re-centred to [-L/2, L/2] when painted (periodic wrap puts negatives in the upper half)"""
        self.attrs['BoxSize'] = numpy.ones(3) * BoxSize
        self.attrs['BoxCenter'] = numpy.ones(3) * BoxCenter

    def to_real_field(self):
        """the FKP field; attrs: data.W, randoms.W, alpha, per-species N / W / W2 / num_per_cell"""
        attrs = {}
        for name in self.source.species:
            attrs[name + '.W'] = self.weighted_total(name)
        attrs['alpha'] = attrs['data.W'] / attrs['randoms.W'] if attrs['randoms.W'] != 0 else numpy.inf
        real = self['data'].to_real_field(normalize=False)
        real.attrs.update(attrs_to_dict(real, 'data.'))
        if self.comm.rank == 0:
            self.logger.info("data painted.")
        if self.source['randoms'].csize > 0:
            real2 = self['randoms'].to_real_field(normalize=False)
            if self.comm.rank == 0:
                self.logger.info("randoms painted.")
            real.axpy(real2, -1. * attrs['alpha'])          # real += (-alpha) * randoms, one pass
            real.attrs.update(attrs_to_dict(real2, 'randoms.'))
            del real2
        vol_per_cell = (self.pm.BoxSize / self.pm.Nmesh).prod()
        real /= vol_per_cell
        if self.comm.rank == 0:
            self.logger.info("volume per cell is %g" % vol_per_cell)
        real.attrs.update(attrs)
        real.attrs.pop('data.shotnoise', None)
        real.attrs.pop('randoms.shotnoise', None)
        return real

    def RecenteredPosition(self, name):
        assert name in ['data', 'randoms']
        return self.source[name][self._uncentered_position] - self.attrs['BoxCenter']

    def TotalWeight(self, name):
        """completeness weight x FKP weight"""
        assert name in ['data', 'randoms']
        return self.source[name][self.comp_weight] * self.source[name][self.fkp_weight]

    def weighted_total(self, name):
        """W = sum of the completeness weights of the selected objects (allreduced)"""
        cat = self.source[name]
        sel = cat[self.selection]
        w = cat[self.comp_weight]
        if not (isinstance(sel, ConstantColumn) and bool(sel.value)):
            w = w[sel]
        return self.comm.allreduce(float(w.sum()))
