"""
FFTPower mode '1d' with the x pass of the r2c fused into the binning (nbk_fft_x_power_bin) against the general path on
the same mesh: the complete field (CatalogMesh.to_complex_field) binned by nbk_power_bin.  Mode counts bit-identical,
k and P within 1e-12 relative per bin (the same per-mode values, summed in another order).
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

RTOL = 1e-12


def _mesh(nmesh, dtype, resampler, box=(600., 500., 400.)):
    from nbodykit_b200.lab import UniformCatalog
    cat = UniformCatalog(nbar=2e5 / np.prod(box), BoxSize=list(box), seed=7)
    return cat.to_mesh(Nmesh=list(nmesh), resampler=resampler, compensated=True, dtype=dtype)


def _edges(mesh, dk):
    box = np.asarray(mesh.attrs['BoxSize'], dtype='f8')
    nmesh = np.asarray(mesh.attrs['Nmesh'])
    kf = 2 * np.pi / box.min()
    dk = kf * dk
    kedges = np.arange(0., np.pi * nmesh.min() / box.max() + dk / 2, dk)
    return [kedges, np.linspace(-1, 1, 2)]


def _bin(field, edges, mesh, comp):
    from nbodykit_b200.algorithms.fftpower import project_to_basis_device
    vol = float(np.prod(mesh.attrs['BoxSize']))
    res, _ = project_to_basis_device(field, edges, los=[0, 0, 1], is_p3d=False, volume=vol,
                                     compensation=(comp, comp), need_mu=False)
    return res


def _check(fused, ref):
    k, _, P, N = fused
    k0, _, P0, N0 = ref
    assert np.array_equal(N, N0)
    np.testing.assert_allclose(k, k0, rtol=RTOL, equal_nan=True)
    assert np.array_equal(np.isnan(P.real), np.isnan(P0.real))
    np.testing.assert_allclose(np.nan_to_num(P.real), np.nan_to_num(P0.real), rtol=RTOL)
    assert not np.any(np.nan_to_num(P.imag)) and not np.any(np.nan_to_num(P0.imag))


def _run(nmesh, dtype, resampler, dk, expect_fused=True):
    mesh = _mesh(nmesh, dtype, resampler)
    comp = mesh._get_compensation()[0][1].__name__
    edges = _edges(mesh, dk)
    # one paint for both paths
    painted, N, W, W2 = mesh._paint_raw()
    nbar = mesh._attrs_for(N, W, W2)[1]
    ref = _bin(painted.r2c(scale=1.0 / nbar), edges, mesh, comp)
    part = painted._r2c_zy()
    part._x_scale = 1.0 / nbar
    fused = _bin(part, edges, mesh, comp)
    # the fused kernel leaves the partial field as it was; the fall-back completes it first
    assert (part._x_scale is not None) == expect_fused
    _check(fused, ref)


@pytest.mark.parametrize("nmesh,resampler", [
    ((256, 256, 256), "cic"), ((256, 256, 256), "tsc"), ((512, 512, 512), "tsc"), ((512, 512, 512), "cic"),
    ((256, 32, 64), "cic"), ((512, 64, 16), "tsc"), ((1024, 16, 8), "tsc"), ((1024, 8, 32), "cic"),
    ((256, 4, 4), "cic"),        # Ny * Nzc = 12 columns: the last tile holds 4 of its 8
])
def test_fused_matches_general_path(cuda, nmesh, resampler):
    _run(nmesh, "f8", resampler, 1.0)


def test_fused_1024_cubed(cuda):
    _run((1024, 1024, 1024), "f8", "cic", 1.0)


@pytest.mark.parametrize("dk,expect_fused", [(0.25, True), (0.05, False)])
def test_many_bins(cuda, dk, expect_fused):
    """k bins beyond what the fused kernel keeps in shared memory take the x pass and nbk_power_bin instead"""
    _run((256, 256, 256), "f8", "cic", dk, expect_fused)


def test_f4_mesh_keeps_the_complete_transform(cuda):
    mesh = _mesh((256, 256, 256), "f4", "cic")
    assert mesh._paint_raw()[0]._r2c_zy() is None


def _spy(monkeypatch):
    """record the fused flag of every nbk_fft_x_power_bin call"""
    from nbodykit_b200 import _lib
    L = _lib.lib()
    orig = L.nbk_fft_x_power_bin
    flags = []

    def spy(*args):
        rc = orig(*args)
        flags.append(args[-2]._obj.value)
        return rc
    monkeypatch.setattr(L, "nbk_fft_x_power_bin", spy)
    return flags


def test_fftpower_1d_takes_fused_path(cuda, monkeypatch):
    """FFTPower mode '1d' on an f8 mesh runs the fused kernel and gives what the general path gives"""
    from nbodykit_b200.lab import FFTPower
    flags = _spy(monkeypatch)
    mesh = _mesh((256, 256, 256), "f8", "cic")
    r = FFTPower(mesh, mode='1d')
    assert flags == [1]
    comp = mesh._get_compensation()[0][1].__name__
    ref = _bin(mesh.to_complex_field(), [r.power.edges['k'], np.linspace(-1, 1, 2)], mesh, comp)
    assert np.array_equal(r.power['modes'], np.squeeze(ref[3]))
    np.testing.assert_allclose(r.power['k'], np.squeeze(ref[0]), rtol=RTOL, equal_nan=True)
    np.testing.assert_allclose(np.nan_to_num(r.power['power'].real), np.nan_to_num(np.squeeze(ref[2]).real), rtol=RTOL)


@pytest.mark.parametrize("mode,dtype", [("2d", "f8"), ("1d", "f4")])
def test_fftpower_other_cases_keep_general_path(cuda, monkeypatch, mode, dtype):
    from nbodykit_b200.lab import FFTPower
    flags = _spy(monkeypatch)
    FFTPower(_mesh((256, 256, 256), dtype, "cic"), mode=mode, Nmu=5)
    assert flags == []
