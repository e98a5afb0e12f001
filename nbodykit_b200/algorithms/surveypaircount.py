"""
Pair counts and two-point correlation functions of survey catalogues (API of
nbodykit/algorithms/pair_counters/mocksurvey.py and paircount_tpcf/tpcf.py: SurveyDataPairCount, SurveyData2PCF) on
one or several GPUs.

The reference converts RA, Dec and redshift to Cartesian positions and hands them to Corrfunc's mocks counters; here
the rows come from transform.SkyToCartesian (or SkyToUnitSphere for 'angular') and are counted by csrc/paircount.cu
under the contract of DESIGN.md 4.8: the observer at the origin, s = x2 - x1 and l = x1 + x2 per axis, the pair's
line of sight along l.  '2d' bins (s, mu = |s.l| / (|s| |l|)), 'projected' bins (r_p, pi = |s.l| / |l|) with
r_p^2 = max(s^2 - pi^2, 0), and 'angular' bins the chord between unit vectors against the chords of the theta edges,
reporting the mean theta in degrees.  '1d' is the non-periodic box count on the Cartesian rows.

Several GPUs: equal-width x slabs of the rows' Cartesian extent, routed as for SimulationBoxPairCount.
"""
import logging

import numpy
import torch

from .._lib import stage
from ..binned_statistic import BinnedStatistic
from ..transform import SkyToCartesian, SkyToUnitSphere
from .fof import _column
from .paircount import (BasePairCount, BasePairCount2PCF, _check_rows, _dims_edges, _smax, _verify_columns, _wedge,
                        check_pair_args, count_pairs, landy_szalay, projected_wp, reduce_histograms, slab_route,
                        weight_column)

_MODE_NAMES = ['1d', '2d', 'projected', 'angular']


def _survey_dims_edges(mode, edges, Nmu, pimax):
    if mode == 'angular':
        return ['theta'], [edges]
    return _dims_edges(mode, edges, Nmu, pimax)


def chord_edges(theta):
    """the chords 2 sin(theta / 2) between unit vectors theta degrees apart: the 'angular' bin edges of the kernel"""
    return 2. * numpy.sin(0.5 * numpy.deg2rad(numpy.asarray(theta, dtype='f8')))


def sky_rows(source, ra, dec, redshift, cosmo, comm, what):
    """float64 device rows of a catalogue's sky columns: SkyToCartesian, or SkyToUnitSphere when ``redshift`` is
    None; RA, Dec and redshift must be finite and redshifts above -1 on every rank (checked on all ranks together, so
    that they raise together)"""
    cols = [_column(source, ra, None)]
    cols.append(_column(source, dec, cols[0].device))
    if redshift is not None:
        cols.append(_column(source, redshift, cols[0].device))
    bad = sum(int((~torch.isfinite(c)).sum().item()) for c in cols)
    if redshift is not None:
        bad += int((cols[2] <= -1).sum().item())
    if comm.allreduce(bad):
        raise ValueError("%s: RA, Dec and redshift must be finite, and redshifts above -1" % what)
    if redshift is None:
        pos = SkyToUnitSphere(cols[0], cols[1])
    else:
        pos = SkyToCartesian(cols[0], cols[1], cols[2], cosmo)
    return pos.contiguous()


class SurveyDataPairCount(BasePairCount):
    r"""
    Count (weighted) pairs of objects of a survey catalogue as a function of :math:`r`, :math:`(r, \mu)`,
    :math:`(r_p, \pi)` or :math:`\theta`, on one or several GPUs.  Runs on construction.

    Parameters
    ----------
    mode : '1d', '2d', 'projected', 'angular'
        bin in the separation, in (separation, mu), in (r_p, pi) or in the angle on the sky
    first : CatalogSource
        the primary catalogue, with RA and Dec in degrees and (unless 'angular') redshift columns
    edges : array_like
        the separation, r_p (Mpc/h) or theta (degrees, at most 180) bin edges, positive, finite and strictly increasing
    cosmo : Cosmology, optional
        converts redshift into comoving distance (any object with ``comoving_distance(z)``); required unless 'angular'
    second : CatalogSource, optional
        the catalogue to cross-correlate with; None (or ``first``) counts the auto pairs
    Nmu : int, optional
        mu bins over [0, 1] ('2d' only)
    pimax : float, optional
        the largest line-of-sight separation ('projected' only); pi bins are ``linspace(0, pimax, int(pimax + 1))``
    ra, dec, redshift, weight : str, optional
        the column names; each pair counts ``w_i * w_j`` in ``wnpairs``
    show_progress, domain_factor, **config :
        recorded in :attr:`attrs`; they have no effect (there is no Corrfunc call or load balancer to pass them to)

    The observer is at the origin and the line of sight of a pair is its midpoint (DESIGN.md 4.8).  Pairs are
    ordered, as Corrfunc counts them: an auto count holds (i, j) and (j, i).  At most 2^31 - 1 rows of each catalogue
    per rank.

    Attributes
    ----------
    pairs : BinnedStatistic
        dims ``['r']``, ``['r', 'mu']``, ``['rp', 'pi']`` or ``['theta']``; variables ``r`` / ``rp`` / ``theta``
        (unweighted mean separation of the pairs in the bin, 0 when empty), ``npairs`` (u8) and ``wnpairs``
    """
    logger = logging.getLogger('SurveyDataPairCount')

    def __init__(self, mode, first, edges, cosmo=None, second=None, Nmu=None, pimax=None, ra='RA', dec='DEC',
                 redshift='Redshift', weight='Weight', show_progress=False, domain_factor=4, **config):
        required = [ra, dec, weight]
        if mode != 'angular':
            required.append(redshift)
        _verify_columns(first, second, required)
        e = check_pair_args(mode, edges, Nmu, pimax)
        if mode == 'angular' and e[-1] > 180.:
            raise ValueError("angular pair count: theta edges are in degrees and may not exceed 180")
        if mode != 'angular' and cosmo is None:
            raise ValueError("'cosmo' keyword is required when 'mode' is not 'angular'")

        self.first = first
        self.second = second
        self.comm = first.comm
        self.attrs = {}
        self.attrs['mode'] = mode
        self.attrs['edges'] = edges
        self.attrs['Nmu'] = Nmu
        self.attrs['pimax'] = pimax
        self.attrs['show_progress'] = show_progress
        self.attrs['N1'] = first.csize
        self.attrs['N2'] = second.csize if second is not None else None
        self.attrs['cosmo'] = cosmo
        self.attrs['weight'] = weight
        self.attrs['ra'] = ra
        self.attrs['dec'] = dec
        self.attrs['redshift'] = redshift
        self.attrs['config'] = config
        self.attrs['domain_factor'] = domain_factor
        self.run()

    def _rows(self, source):
        a = self.attrs
        z = None if a['mode'] == 'angular' else a['redshift']
        with stage("paircount_sky"):
            pos = sky_rows(source, a['ra'], a['dec'], z, a['cosmo'], self.comm, "SurveyDataPairCount")
            return pos, weight_column(source, a['weight']).to(pos.device)

    def run(self):
        """count the pairs; sets :attr:`pairs` and ``attrs['total_wnpairs']`` / ``attrs['is_cross']``"""
        comm = self.comm
        attrs = self.attrs
        mode = attrs['mode']
        auto = self.second is None or self.second is self.first
        pos1, w1 = self._rows(self.first)
        pos2, w2 = (pos1, w1) if auto else self._rows(self.second)
        _check_rows(int(pos1.shape[0]), "the first catalogue")
        _check_rows(int(pos2.shape[0]), "the second catalogue")

        # the normalisation of the estimators (0.5 by convention; it cancels in every ratio)
        s1 = comm.allreduce(float(w1.sum().item()))
        if auto:
            s2 = comm.allreduce(float((w1 * w1).sum().item()))
            attrs['total_wnpairs'] = 0.5 * (s1 ** 2 - s2)
            attrs['is_cross'] = False
        else:
            s2 = comm.allreduce(float(w2.sum().item()))
            attrs['total_wnpairs'] = 0.5 * s1 * s2
            attrs['is_cross'] = True

        e = numpy.asarray(attrs['edges'], dtype='f8')
        kedges = chord_edges(e) if mode == 'angular' else e
        smax = _smax(mode, kedges, attrs['pimax'])
        with stage("paircount_route"):
            if comm.size > 1:
                pos1, w1, pos2, w2 = slab_route(comm, pos1, w1, pos2, w2, False, None, smax)
                _check_rows(int(pos1.shape[0]), "primaries after routing")
                _check_rows(int(pos2.shape[0]), "secondaries after routing")
        npairs, wsum, ssum, cand = count_pairs(mode, pos1, w1, pos2, w2, kedges, False, None, 2, attrs['Nmu'],
                                               attrs['pimax'], survey=True)
        with stage("paircount_reduce"):
            npairs, wsum, ssum, cand = reduce_histograms(comm, npairs, wsum, ssum, cand)
        self.candidates = cand

        dims, edges = _survey_dims_edges(mode, attrs['edges'], attrs['Nmu'], attrs['pimax'])
        shape = tuple(len(x) - 1 for x in edges)
        data = numpy.zeros(shape, dtype=[(dims[0], 'f8'), ('npairs', 'u8'), ('wnpairs', 'f8')])
        n = npairs.reshape(shape)
        data['npairs'] = n
        data['wnpairs'] = wsum.reshape(shape)
        sep = numpy.zeros(shape)
        numpy.divide(ssum.reshape(shape), n, out=sep, where=n > 0)
        data[dims[0]] = sep
        self.pairs = BinnedStatistic(dims, edges, data, fields_to_sum=['npairs', 'wnpairs'])
        self.pairs.attrs['total_wnpairs'] = attrs['total_wnpairs']

    # ------------------------------------------------------------------------------------------------------------------
    def __setstate__(self, state):
        self.__dict__.update(state)
        a = self.attrs
        if a['mode'] not in _MODE_NAMES:
            raise ValueError("mode = '%s' should be one of %s" % (a['mode'], _MODE_NAMES))
        dims, edges = _survey_dims_edges(a['mode'], a['edges'], a['Nmu'], a['pimax'])
        self.pairs = BinnedStatistic(dims, edges, self.pairs, fields_to_sum=['npairs', 'wnpairs'])


class SurveyData2PCF(BasePairCount2PCF):
    r"""
    The two-point correlation function of survey catalogues, from pair counts, as a function of :math:`r`,
    :math:`(r, \mu)`, :math:`(r_p, \pi)` or :math:`\theta`, with the Landy-Szalay estimator.  Runs on construction.

    ``randoms2`` defaults to ``randoms1`` when ``data2`` is given; a given ``R1R2`` (a :class:`SurveyDataPairCount`)
    is used instead of counting the random pairs.  The other parameters are those of :class:`SurveyDataPairCount`.

    Attributes
    ----------
    D1D2, D1R2, D2R1, R1R2 : WedgeBinnedStatistic
        the pair counts
    corr : WedgeBinnedStatistic
        the correlation function (``corr``) and the mean separation of the D1D2 pairs
    wp : WedgeBinnedStatistic
        ``'projected'`` only: :math:`w_p(r_p) = 2 \sum \xi \Delta\pi` in ``corr``
    """
    logger = logging.getLogger('SurveyData2PCF')

    def __init__(self, mode, data1, randoms1, edges, cosmo=None, Nmu=None, pimax=None, data2=None, randoms2=None,
                 R1R2=None, ra='RA', dec='DEC', redshift='Redshift', weight='Weight', show_progress=False, **config):
        self.comm = data1.comm
        self.attrs = {'mode': mode, 'edges': numpy.array(edges), 'Nmu': Nmu, 'pimax': pimax, 'cosmo': cosmo, 'ra': ra,
                      'dec': dec, 'redshift': redshift, 'weight': weight, 'show_progress': show_progress,
                      'config': config}
        self.data1, self.data2 = data1, data2
        self.randoms1, self.randoms2 = randoms1, randoms2
        self.R1R2 = R1R2
        self.run()

    def run(self):
        """count the pairs and apply the estimator; sets D1D2, D1R2, D2R1, R1R2, corr (and wp)"""
        kw = dict(self.attrs)
        kw.update(kw.pop('config'))
        if self.randoms1 is None:
            raise ValueError("a catalog of randoms must be specified as the ``randoms1`` keyword for survey data")
        if self.data2 is not None and self.randoms2 is None:
            self.randoms2 = self.randoms1
        r2 = self.randoms2 if self.randoms2 is not None else self.randoms1
        RR = self.R1R2
        if RR is None:
            RR = SurveyDataPairCount(first=self.randoms1, second=r2, **kw)
        DD = SurveyDataPairCount(first=self.data1, second=self.data2, **kw)
        DR = SurveyDataPairCount(first=self.data1, second=r2, **kw)
        RD = SurveyDataPairCount(first=self.data2, second=self.randoms1, **kw) if self.data2 is not None else DR
        self.corr = landy_szalay(DD, DR, RD, RR)
        self.D1D2, self.D1R2, self.D2R1, self.R1R2 = DD.pairs, DR.pairs, RD.pairs, RR.pairs
        for name in ('D1D2', 'D1R2', 'D2R1', 'R1R2'):
            setattr(self, name, _wedge(getattr(self, name)))
        self.wp = projected_wp(self.corr) if self.attrs['mode'] == 'projected' else None
