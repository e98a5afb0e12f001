"""Host-side logic of the nbodykit API layer that needs no GPU."""
import json

import numpy as np
import pytest

from nbodykit_b200 import CurrentMPIComm, set_options, _global_options
from nbodykit_b200.base.catalog import Column, ConstantColumn
from nbodykit_b200.comm import SelfComm
from nbodykit_b200.lab import ArrayCatalog, UniformCatalog, RandomCatalog, FFTPower
from nbodykit_b200.mpirng import MPIRandomState
from nbodykit_b200.utils import JSONDecoder, JSONEncoder


def test_options_context():
    assert _global_options['paint_chunk_size'] == 4 * 1024 * 1024
    with set_options(paint_chunk_size=123):
        assert _global_options['paint_chunk_size'] == 123
    assert _global_options['paint_chunk_size'] == 4 * 1024 * 1024
    with pytest.raises(KeyError):
        set_options(nonsense=1)


def test_current_comm_stack():
    c = CurrentMPIComm.get()
    assert c.rank == 0 and c.size == 1
    other = SelfComm()
    with CurrentMPIComm.enter(other):
        assert CurrentMPIComm.get() is other
        cat = UniformCatalog(nbar=10, BoxSize=1., seed=1)
        assert cat.comm is other
    assert CurrentMPIComm.get() is c


def test_uniform_catalog_columns_and_attrs():
    cat = UniformCatalog(nbar=100, BoxSize=[1., 2., 3.], seed=42)
    assert cat.attrs['seed'] == 42 and list(cat.attrs['BoxSize']) == [1., 2., 3.]
    assert cat.columns == ['Position', 'Selection', 'Value', 'Velocity', 'Weight']
    pos = cat['Position'].compute()
    assert pos.shape == (cat.size, 3) and pos.dtype == np.float64
    assert (pos >= 0).all() and (pos <= [1., 2., 3.]).all()
    # default columns are never materialised
    assert isinstance(cat['Weight'], ConstantColumn) and cat['Weight'].value == 1.0
    assert isinstance(cat['Selection'], ConstantColumn) and cat['Selection'].value is True
    with pytest.raises(ValueError):
        UniformCatalog(nbar=1e-9, BoxSize=1., seed=1)
    f4 = UniformCatalog(nbar=100, BoxSize=1., seed=42, dtype='f4')
    assert f4['Position'].dtype == np.float32


def test_column_protocol():
    cat = UniformCatalog(nbar=1000, BoxSize=1., seed=3)
    n = cat.size
    cat['Mass'] = np.arange(n, dtype='f8')
    cat['Flag'] = 2.5
    assert 'Mass' in cat and isinstance(cat['Flag'], ConstantColumn)
    with pytest.raises(ValueError):
        cat['Bad'] = np.arange(n + 1)
    with pytest.raises(KeyError):
        cat['Nope']
    sub = cat[cat['Mass'] < 10]
    assert sub.size == 10 and sub['Flag'].value == 2.5 and sub.attrs['seed'] == 3
    np.testing.assert_array_equal(sub['Mass'].compute(), np.arange(10.))
    sl = cat[5:15]
    assert sl.size == 10 and sl['Mass'].compute()[0] == 5
    only = cat[['Position', 'Mass']]
    assert only.columns == ['Mass', 'Position', 'Selection', 'Value', 'Weight']
    rsd = cat['Position'] + cat['Velocity'] * [0, 0, 1]
    assert isinstance(rsd, Column) and rsd.shape == (n, 3)
    np.testing.assert_allclose(rsd.compute()[:, 2], cat['Position'].compute()[:, 2] + cat['Velocity'].compute()[:, 2])
    p, m = cat.compute(cat['Position'], cat['Mass'])
    assert p.shape == (n, 3) and m.shape == (n,)
    del cat['Mass']
    assert 'Mass' not in cat


def test_array_catalog():
    data = np.zeros(10, dtype=[('Position', ('f4', 3)), ('Mass', 'f8')])
    cat = ArrayCatalog(data, BoxSize=5.)
    assert cat.size == 10 and cat.csize == 10 and cat.attrs['BoxSize'] == 5.
    assert 'Mass' in cat and 'Weight' in cat
    with pytest.raises(ValueError):
        ArrayCatalog(np.zeros(3))
    with pytest.raises(ValueError):
        ArrayCatalog({'a': np.zeros(3), 'b': np.zeros(4)})


def test_to_mesh_argument_errors():
    cat = ArrayCatalog({'Position': np.zeros((4, 3))})
    with pytest.raises(ValueError):
        cat.to_mesh(Nmesh=8)                       # no BoxSize anywhere
    with pytest.raises(ValueError):
        cat.to_mesh(BoxSize=1.)                    # no Nmesh anywhere
    with pytest.raises(ValueError):
        cat.to_mesh(Nmesh=8, BoxSize=1., resampler='nope')
    with pytest.raises(ValueError):
        cat.to_mesh(Nmesh=8, BoxSize=1., weight='nope')
    mesh = cat.to_mesh(Nmesh=8, BoxSize=1., resampler='db6')      # name accepted ...
    mesh.compensated = True
    with pytest.raises(ValueError):
        mesh.actions                               # ... but no compensation defined (test_catalogmesh.py:133-145)
    mesh = cat.to_mesh(Nmesh=8, BoxSize=1., resampler='tsc', interlaced=True, compensated=True)
    assert mesh.attrs['resampler'] == 'tsc' and mesh.interlaced and mesh.compensated
    assert mesh.actions[0][1].__name__ == 'CompensateTSC' and mesh.actions[0][2] == 'circular'
    mesh.interlaced = False
    assert mesh.actions[0][1].__name__ == 'CompensateTSCShotnoise'
    assert len(mesh) == 0
    with pytest.raises(AssertionError):
        mesh.resampler = 'nope'


def test_fftpower_argument_errors():
    cat = ArrayCatalog({'Position': np.zeros((4, 3))}, BoxSize=1.)
    with pytest.raises(ValueError):
        FFTPower(cat, mode='3d', Nmesh=8)
    with pytest.raises(ValueError):
        FFTPower(cat, mode='1d', Nmesh=8, los=[0, 0, 2])
    with pytest.raises(ValueError):
        FFTPower(cat, mode='1d', Nmesh=8, los=1)
    with pytest.raises(TypeError):
        FFTPower(object(), mode='1d', Nmesh=8)


def test_mesh_actions_view():
    from nbodykit_b200.base.mesh import MeshFilter
    cat = ArrayCatalog({'Position': np.zeros((4, 3))}, BoxSize=1.)
    mesh = cat.to_mesh(Nmesh=8)
    f = lambda k, v: v
    view = mesh.apply(f, kind='wavenumber', mode='complex')
    assert view is not mesh and view.actions[-1] == ('complex', f, 'wavenumber') and mesh.actions == []
    with pytest.raises(AssertionError):
        mesh.apply(f, kind='relative', mode='complex')

    class Flt(MeshFilter):
        kind = 'circular'
        mode = 'complex'

        def filter(self, k, v):
            return v
    assert mesh.apply(Flt).actions[-1][2] == 'circular'


def test_json_encoder_matches_reference_wire_format():
    arr = np.zeros(2, dtype=[('k', 'f8'), ('power', 'c16'), ('modes', 'i8')])
    arr['power'] = [1 + 2j, 3 - 1j]
    s = json.dumps(dict(a=arr, b=np.float32(1.5), c=np.int64(3), d=2 + 1j, e=np.arange(3.)), cls=JSONEncoder)
    raw = json.loads(s)
    assert raw['a']['__dtype__'] == [['k', '<f8'], ['power', '<c16'], ['modes', '<i8']]
    assert raw['a']['__shape__'] == [2] and raw['a']['__data__'][0][1] == {'__complex__': [1.0, 2.0]}
    assert raw['d'] == {'__complex__': [2.0, 1.0]} and raw['b'] == 1.5 and raw['c'] == 3
    back = json.loads(s, cls=JSONDecoder)
    np.testing.assert_array_equal(back['a'], arr)
    assert back['d'] == 2 + 1j
    np.testing.assert_array_equal(back['e'], np.arange(3.))


class _FakeRankComm(object):
    """deterministic stand-in for one rank of an n-rank communicator (sizes known up front)"""

    def __init__(self, rank, sizes):
        self.rank, self.size, self._sizes = rank, len(sizes), sizes

    def allgather(self, x):
        assert not isinstance(x, np.ndarray)
        return list(self._sizes)

    def allreduce(self, x, op=None):
        return sum(self._sizes)


@pytest.mark.parametrize("sizes", [[250001], [100000, 150001], [1, 99999, 100000, 50001], [0, 250001], [33333, 0, 216668]])
def test_mpirng_is_rank_count_invariant(sizes):
    """nbodykit/tests/test_mpirng.py:12-90: the gathered result equals the single-rank result"""
    full = MPIRandomState(SelfComm(), seed=5, size=sum(sizes))
    want_u = full.uniform(itemshape=(3,))
    want_n = full.normal(loc=2.)
    got_u, got_n = [], []
    for r in range(len(sizes)):
        rng = MPIRandomState(_FakeRankComm(r, sizes), seed=5, size=sizes[r])
        got_u.append(rng.uniform(itemshape=(3,)))
        got_n.append(rng.normal(loc=2.))
    np.testing.assert_array_equal(np.concatenate(got_u), want_u)
    np.testing.assert_array_equal(np.concatenate(got_n), want_n)


def test_random_catalog():
    cat = RandomCatalog(1000, seed=2)
    assert cat.size == 1000 and cat.attrs['seed'] == 2
    cat['z'] = cat.rng.normal(loc=0.5, scale=0.1)
    assert abs(cat['z'].compute().mean() - 0.5) < 0.02
    with pytest.raises(ValueError):
        RandomCatalog(0, seed=1)


def test_find_unique_edges_matches_reference_formula():
    """dk=0 unique-|k| edges from 1-D coordinates only == the reference's full-array procedure"""
    from nbodykit_b200.algorithms.fftpower import _find_unique_edges
    from nbodykit_b200.pmesh.pm import ParticleMesh
    from oracle import pmesh_oracle as po
    N, L = 8, 10.
    pm = ParticleMesh(BoxSize=L, Nmesh=N, dtype='f8', comm=SelfComm())
    kmax = np.pi * N / L + 1e-9
    edges, centers = _find_unique_edges(pm, kmax)
    x = po.k_coords(N, L, "f4")
    fx2 = (0 + x[0] ** 2 + x[1] ** 2 + x[2] ** 2).ravel()
    binning = (2 * np.pi / L * 0.05) ** 2
    ix2 = np.int64(fx2 / binning + 0.5)
    _, ind = np.unique(ix2, return_index=True)
    fx = fx2[ind] ** 0.5
    fx = fx[fx < kmax]
    np.testing.assert_array_equal(centers, fx)
    assert edges[0] == 0 and len(edges) == len(centers) + 1 and np.all(np.diff(edges) > 0)


def test_fftrecon_and_projected_power_argument_checks():
    """host-side validation mirrors the reference (fftrecon.py:76-129, fftpower.py:393-399); nothing touches the GPU"""
    import warnings
    from nbodykit_b200.lab import ArrayCatalog, FFTRecon, ProjectedFFTPower
    rng = np.random.RandomState(0)
    d = ArrayCatalog({'Position': rng.uniform(0, 100., size=(50, 3)), 'Other': np.zeros(50)}, BoxSize=100., Nmesh=8)
    r = ArrayCatalog({'Position': rng.uniform(0, 100., size=(80, 3))}, BoxSize=100.)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = FFTRecon(data=d, ran=r, Nmesh=None, bias=2.0, f=0.5, los=[0, 0, 2], R=20., scheme='LF2')
    assert list(m.attrs['Nmesh']) == [8, 8, 8] and list(m.attrs['BoxSize']) == [100., 100., 100.]
    np.testing.assert_allclose(m.attrs['los'], [0, 0, 0.5])          # los / sum(los^2), as the reference does
    assert m.attrs['scheme'] == 'LF2' and m.attrs['revert_rsd_random'] is False and m.dtype == 'f8'
    with pytest.raises(AssertionError):
        FFTRecon(data=d, ran=r, Nmesh=8, scheme='XYZ')
    with pytest.raises(AssertionError):
        FFTRecon(data=d, ran=r, Nmesh=8, position='Other')            # the randoms have no such column
    with pytest.warns(UserWarning):
        FFTRecon(data=d, ran=r, Nmesh=8, R=1.0)                       # smoothing below the cell size
    with pytest.raises(AssertionError):
        ProjectedFFTPower(d, Nmesh=8, axes=(0, 1, 2))


def test_push_chunks_clamp():
    """parts the slab exchange of the distributed r2c is pipelined in: 4, bounded by the planes of the slab"""
    from nbodykit_b200.pmesh.pm import _push_chunks
    assert _push_chunks(128) == 4 and _push_chunks(2) == 2 and _push_chunks(1) == 1
