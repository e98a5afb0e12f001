"""ConvolvedFFT3PCF without a GPU: the oracle's FFT form (scipy Y_lm, rfftn) equals its direct form (every true
separation, explicit Legendre polynomials) on fields the geometry guard accepts; threeptcf.edge_correct (the closed-form
3j symbols, a planted zeta, the Legendre product of zeta and R by quadrature, M = I, NaN where rrr_0 = 0); the window
box; every argument and geometry error is raised before any paint or
transform; the transform count and blocks; the table layout; save / load."""
import numpy as np
import pytest

import convfft3pcf_oracle as cfo

POLES = [0, 1, 2, 3, 4]


def _padded(N, box, seed):
    """a skewed field that is zero outside the cells box = (lo, hi) per axis"""
    rng = np.random.RandomState(seed)
    F = np.zeros(N)
    sl = tuple(slice(a, b) for a, b in box)
    g = rng.standard_normal(F[sl].shape)
    F[sl] = g + 0.5 * g ** 2
    return F


@pytest.mark.parametrize("N,L,box,edges", [
    ((12, 12, 12), (120., 120., 120.), ((2, 7), (3, 8), (1, 6)), [0., 14., 27., 41., 55.]),
    ((12, 10, 9), (130., 100., 90.), ((0, 5), (4, 9), (2, 6)), [5., 17., 30., 44.]),
])
def test_fft_form_equals_direct_form(N, L, box, edges):
    # the fields span at most 5 cells per axis, so with max(edges) below L - 5 H no pair wraps
    Nf = _padded(N, box, 1) - 0.4 * _padded(N, box, 2)
    Rf = np.abs(_padded(N, box, 3)) + 0.1
    Rf[Nf == 0] = 0
    a = cfo.fft_form(Nf, Rf, N, L, edges, POLES)
    b = cfo.direct_form(Nf, Rf, N, L, edges, POLES)
    assert (a["nsep"] > 0).all()
    for k, bound in (("nnn", "bound_n"), ("rrr", "bound_r")):
        err = np.abs(a[k] - b[k]) / a[bound]
        assert err.max() <= 1e-12, (k, err.max())
        # far from zero against the bound: the comparison is not vacuous
        assert (np.abs(a[k][0]) / a[bound][0]).max() > 1e-3
        assert (np.abs(a[k][1:]) / a[bound][1:]).max() > 1e-4


def test_direct_form_sees_no_wrap():
    """a field in one corner: with true separations its pairs across the periodic boundary do not count"""
    N, L = (10, 10, 10), (10., 10., 10.)
    W = np.zeros(N)
    W[0, 0, 0] = W[9, 0, 0] = 1.0                                  # 1 cell apart only through the wrap
    out = cfo.direct_form(W, W, N, L, [0.5, 1.5], [0])
    assert out["nnn"][0, 0, 0] == 0
    W[1, 0, 0] = 1.0
    assert cfo.direct_form(W, W, N, L, [0.5, 1.5], [0])["nnn"][0, 0, 0] > 0


# ---- edge_correct
def test_threej_closed_form_matches_sympy():
    wigner = pytest.importorskip("sympy.physics.wigner")
    from nbodykit_b200.algorithms.threeptcf import threej_squared
    err = 0.
    for a in range(11):
        for b in range(11):
            for c in range(11):
                err = max(err, abs(float(wigner.wigner_3j(a, b, c, 0, 0, 0) ** 2) - float(threej_squared(a, b, c))))
    assert err <= 3e-17, err


def test_threej_closed_form_matches_gauss_legendre():
    """int_{-1}^{1} P_a P_b P_c = 2 (a b c; 0 0 0)^2, by a quadrature exact for the degree"""
    from scipy.special import eval_legendre
    from nbodykit_b200.algorithms.threeptcf import threej_squared
    x, w = np.polynomial.legendre.leggauss(20)
    for a in range(11):
        for b in range(11):
            for c in range(11):
                q = np.sum(w * eval_legendre(a, x) * eval_legendre(b, x) * eval_legendre(c, x))
                assert abs(q - 2 * float(threej_squared(a, b, c))) <= 1e-14, (a, b, c)


def _planted(poles, nb, seed):
    from nbodykit_b200.algorithms.threeptcf import threej_squared
    rng = np.random.RandomState(seed)
    zeta = rng.standard_normal((len(poles), nb, nb))
    r0 = rng.uniform(1., 3., (nb, nb))
    f = 0.3 * rng.standard_normal((len(poles), nb, nb))
    f[poles.index(0)] = 1.
    nnn = np.zeros_like(zeta)
    for a, la in enumerate(poles):
        for c, lc in enumerate(poles):
            for k, lk in enumerate(poles):
                nnn[a] += (2 * la + 1) * float(threej_squared(la, lc, lk)) * zeta[c] * f[k] * r0
    return nnn, f * r0, zeta


@pytest.mark.parametrize("poles", [[0, 1, 2, 3, 4], [3, 0, 2, 1], list(range(11))])
def test_edge_correct_recovers_a_planted_zeta(poles):
    """nnn = RRR times a 3PCF with no multipoles above max(poles), and R none either: the system is exact"""
    from nbodykit_b200.algorithms.threeptcf import edge_correct
    nnn, rrr, zeta = _planted(poles, 4, 7)
    err = np.abs(edge_correct(nnn, rrr, poles) - zeta).max()
    assert err <= 1e-12 * np.abs(zeta).max(), err


def test_edge_correct_is_the_identity_without_window_multipoles():
    """f = delta_l0: M = I, zeta = nnn / rrr_0; NaN where rrr_0 = 0"""
    from nbodykit_b200.algorithms.threeptcf import edge_correct
    rng = np.random.RandomState(3)
    poles = [2, 0, 1]
    nnn = rng.standard_normal((3, 4, 4))
    rrr = np.zeros((3, 4, 4))
    rrr[1] = rng.uniform(1, 2, (4, 4))
    rrr[1, 2, 3] = rrr[1, 3, 2] = 0.
    z = edge_correct(nnn, rrr, poles)
    ok = rrr[1] != 0
    np.testing.assert_allclose(z[:, ok], nnn[:, ok] / rrr[1][ok], rtol=1e-15)
    assert np.isnan(z[:, ~ok]).all() and (~ok).sum() == 2


@pytest.mark.parametrize("poles", [[1, 2], [0, 2], [0, 1, 3]])
def test_edge_correct_refuses_gaps(poles):
    from nbodykit_b200.algorithms.threeptcf import edge_correct
    with pytest.raises(ValueError):
        edge_correct(np.ones((len(poles), 2, 2)), np.ones((len(poles), 2, 2)), poles)


# ---- arguments and geometry, before any paint or transform
def _fkp(C, ext, nd=50, nr=200, empty_randoms=False, seed=0, rsel=None, rweight=None):
    """host columns: data and randoms uniform in a cube of side ext around C, and a far-away data row deselected;
    rsel / rweight: a Selection / Weight value for every random"""
    from nbodykit_b200.lab import ArrayCatalog, FKPCatalog
    rng = np.random.RandomState(seed)
    dpos = rng.uniform(-0.5, 0.5, (nd, 3)) * ext + C
    dpos[0] = C + 1e4                                                 # deselected: outside the bounds
    sel = np.ones(nd, dtype=bool)
    sel[0] = False
    d = ArrayCatalog({"Position": dpos, "NZ": np.ones(nd), "Selection": sel})
    nr = 0 if empty_randoms else nr
    cols = {"Position": rng.uniform(-0.5, 0.5, (nr, 3)) * ext + C, "NZ": np.ones(nr)}
    if rsel is not None:
        cols["Selection"] = np.full(nr, rsel)
    if rweight is not None:
        cols["Weight"] = np.full(nr, rweight)
    r = ArrayCatalog(cols)
    return FKPCatalog(d, r), dpos[1:], r["Position"]


def _stubbed(monkeypatch):
    from nbodykit_b200.algorithms import convfft3pcf
    ran = []
    monkeypatch.setattr(convfft3pcf.ConvolvedFFT3PCF, "run", lambda self: ran.append(self.attrs))
    return convfft3pcf.ConvolvedFFT3PCF, ran


@pytest.mark.parametrize("poles,edges", [
    ([0, 2], [0., 10.]), ([1, 2], [0., 10.]), ([0, 1, 3], [0., 10.]), ([], [0., 10.]), ([0, 0, 1], [0., 10.]),
    ([0, 11], [0., 10.]), ([0, 1.5], [0., 10.]),
    ([0], [10.]), ([0], [10., 5.]), ([0], [-1., 5.]), ([0], [0., np.inf]), ([0], np.linspace(0, 30, 34)),
])
def test_bad_arguments_raise_before_device_work(monkeypatch, poles, edges):
    cls, ran = _stubbed(monkeypatch)
    fkp, _, _ = _fkp(np.array([500., 500., 500.]), 60.)
    mesh = fkp.to_mesh(Nmesh=32, BoxSize=200., BoxCenter=500., dtype="f8", resampler="cic")
    with pytest.raises(ValueError):
        cls(mesh, poles, edges)
    assert not ran


def test_good_arguments_reach_run(monkeypatch):
    cls, ran = _stubbed(monkeypatch)
    fkp, _, _ = _fkp(np.array([500., 500., 500.]), 60.)
    mesh = fkp.to_mesh(Nmesh=32, BoxSize=200., BoxCenter=500., dtype="c16", resampler="tsc", interlaced=True)
    cls(mesh, [2, 0, 1], [0., 20., 40.])
    assert ran and ran[0]["poles"] == [2, 0, 1]
    for key in ("poles", "edges", "Nmesh", "BoxSize", "BoxCenter"):
        assert key in ran[0]
    with pytest.raises(TypeError):
        cls(object(), [0], [0., 10.])


def test_geometry_guard_names_the_box_that_passes(monkeypatch):
    """extent + (support + 2) H + r_max < L per axis: a box just too small raises, naming the smallest BoxSize that
    passes; that BoxSize (a hair above) passes, and the deselected far-away row does not count"""
    from nbodykit_b200.algorithms.convfft3pcf import min_box_size
    cls, ran = _stubbed(monkeypatch)
    C = np.array([500., -200., 30.])
    fkp, dpos, rpos = _fkp(C, 60.)
    allpos = np.concatenate([dpos, rpos])
    lo, hi = allpos.min(0) - C, allpos.max(0) - C
    N, rmax, support = 32, 40., 3                                # tsc
    need = min_box_size(lo, hi, [N] * 3, support, rmax)
    np.testing.assert_allclose(need, ((hi - lo) + rmax) / (1 - (support + 2) / N), rtol=1e-15)
    edges = [0., 20., rmax]
    small = float(need.max()) * 0.999
    mesh = fkp.to_mesh(Nmesh=N, BoxSize=small, BoxCenter=C, dtype="f8", resampler="tsc", interlaced=True)
    with pytest.raises(ValueError) as exc:
        cls(mesh, [0, 1], edges)
    assert "[%s]" % ", ".join("%.6g" % x for x in need) in str(exc.value)
    assert not ran
    mesh = fkp.to_mesh(Nmesh=N, BoxSize=float(need.max()) * 1.0001, BoxCenter=C, dtype="f8", resampler="tsc",
                       interlaced=True)
    cls(mesh, [0, 1], edges)
    assert len(ran) == 1


def test_rmax_above_half_the_box_raises(monkeypatch):
    """a tiny survey in a large box still needs r_max <= L / 2: the message names 2 r_max"""
    cls, ran = _stubbed(monkeypatch)
    C = np.zeros(3)
    fkp, _, _ = _fkp(C, 1.)
    mesh = fkp.to_mesh(Nmesh=64, BoxSize=[100., 100., 70.], BoxCenter=C, dtype="f8", resampler="cic")
    with pytest.raises(ValueError) as exc:
        cls(mesh, [0], [0., 40.])
    assert "80, 80, 80" in str(exc.value)
    assert not ran


@pytest.mark.parametrize("kw", [dict(empty_randoms=True), dict(rsel=False), dict(rweight=0.)])
def test_empty_randoms_raise(monkeypatch, kw):
    """no randoms, randoms of which none is selected, and selected randoms of zero total weight"""
    cls, ran = _stubbed(monkeypatch)
    fkp, _, _ = _fkp(np.zeros(3), 20., **kw)
    mesh = fkp.to_mesh(Nmesh=32, BoxSize=200., BoxCenter=0., dtype="f8", resampler="cic", bbox_from_species="data")
    with pytest.raises(ValueError, match="ConvolvedFFT3PCF: .*randoms"):
        cls(mesh, [0], [0., 10.])
    assert not ran


def test_window_box_and_mask():
    """the box is the guard's width; a cell is in it when its node, wrapped with period L, lies in [a, b] -- also
    for a box across the index boundary"""
    from nbodykit_b200.algorithms.convfft3pcf import box_mask, window_box
    lo, hi, H = np.array([-7.3, 2., -30.]), np.array([4.1, 9.5, -21.]), np.array([2., 2.5, 4.])
    a, b = window_box(lo, hi, H, 3)
    np.testing.assert_allclose(b - a, (hi - lo) + 5 * H, rtol=1e-15)
    N, L = (16, 20, 25), H * np.array([16, 20, 25])
    for d, m in enumerate(box_mask(N, L, a, b)):
        node = np.arange(N[d]) * H[d]
        want = np.zeros(N[d], dtype=bool)
        for k in (-2, -1, 0, 1):
            want |= (node + k * L[d] >= a[d]) & (node + k * L[d] <= b[d])
        np.testing.assert_array_equal(m.astype(bool), want)
        assert 0 < m.sum() < N[d]
    assert box_mask(N, L, a, b)[0][0] == 1 and box_mask(N, L, a, b)[0][-1] == 1      # across the boundary


def test_edge_correct_against_legendre_quadrature():
    """independent of the coupling formula: zeta(mu) and R(mu) as Legendre series (R with no multipoles above
    max(poles)), N(mu) = zeta(mu) R(mu), and nnn_l / rrr_l their Legendre coefficients (2l + 1) / 2 int P_l by
    Gauss-Legendre quadrature, exact for these degrees"""
    from numpy.polynomial import legendre as leg
    from nbodykit_b200.algorithms.threeptcf import edge_correct
    rng = np.random.RandomState(11)
    for poles in ([0, 1, 2, 3, 4], [4, 2, 0, 3, 1], list(range(11))):
        L = max(poles)
        zc = rng.standard_normal(L + 1)
        rc = np.concatenate([[1.], 0.3 * rng.standard_normal(L)]) * 2.5
        x, w = leg.leggauss(2 * L + 2)
        Nmu = leg.legval(x, zc) * leg.legval(x, rc)
        coef = lambda f, ell: (2 * ell + 1) / 2 * np.sum(w * f * leg.legval(x, np.eye(L + 1)[ell]))   # noqa: E731
        nnn = np.array([coef(Nmu, ell) for ell in poles])[:, None, None]
        rrr = np.array([coef(leg.legval(x, rc), ell) for ell in poles])[:, None, None]
        z = edge_correct(nnn, rrr, poles)[:, 0, 0]
        np.testing.assert_allclose(z, zc[poles], rtol=0, atol=1e-12 * np.abs(zc).max())


# ---- counts, layout, save / load
def test_transform_count_and_blocks():
    from nbodykit_b200.algorithms.fft3pcf import bin_blocks, transform_count
    poles = list(range(11))
    assert transform_count(bin_blocks(8, 8), poles, 2) == 2 + 3 * 8 * 121
    assert transform_count(bin_blocks(8, 8), poles) == 1 + 2 * 8 * 121
    assert transform_count(bin_blocks(6, 3), [0, 1, 2], 2) == 2 + 3 * 9 * (1 * 1 + 1 * 2 + 1 * 3 + 1 * 4 + 1 * 5 + 1 * 6)
    assert transform_count(bin_blocks(8, 5), [0, 2], 2) == 2 + 3 * 6 * (2 + 4 + 6 + 8)


def _table():
    from nbodykit_b200.algorithms.convfft3pcf import pole_table
    rng = np.random.RandomState(4)
    nnn, rrr, zeta = (rng.standard_normal((2, 3, 3)) for _ in range(3))
    return nnn, rrr, zeta, pole_table(nnn, rrr, zeta, [1, 0])


def test_pole_table_layout():
    nnn, rrr, zeta, d = _table()
    assert d.dtype.names == ("nnn_1", "nnn_0", "rrr_1", "rrr_0", "zeta_1", "zeta_0")
    for p, ell in enumerate([1, 0]):
        np.testing.assert_array_equal(d["nnn_%d" % ell], nnn[p])
        np.testing.assert_array_equal(d["rrr_%d" % ell], rrr[p])
        np.testing.assert_array_equal(d["zeta_%d" % ell], zeta[p])


def test_save_load_round_trip(tmp_path):
    from nbodykit_b200.algorithms.convfft3pcf import ConvolvedFFT3PCF
    from nbodykit_b200.binned_statistic import BinnedStatistic
    from nbodykit_b200.comm import SelfComm
    nnn, rrr, zeta, d = _table()
    e = np.array([0., 10., 20., 30.])
    r = object.__new__(ConvolvedFFT3PCF)
    r.comm = SelfComm()
    r.attrs = dict(poles=[1, 0], edges=e, Nmesh=np.array([8, 8, 8]), BoxSize=np.array([60.] * 3),
                   BoxCenter=np.array([1., 2., 3.]), alpha=0.1, transforms=44, tiles=0.25,
                   **{"data.W": 10., "randoms.W": 100.})
    r.nsep = np.array([4, 0, 6], dtype="u8")
    r.poles = BinnedStatistic(["r1", "r2"], [e, e], d)
    path = str(tmp_path / "cf.json")
    r.save(path)
    s = ConvolvedFFT3PCF.load(path, comm=SelfComm())
    assert s.poles.dims == ["r1", "r2"]
    np.testing.assert_array_equal(s.poles.edges["r1"], e)
    for f in d.dtype.names:
        np.testing.assert_array_equal(s.poles[f], r.poles[f])
    np.testing.assert_array_equal(s.nsep, r.nsep)
    assert s.nsep.dtype == np.dtype("u8")
    assert s.attrs["poles"] == [1, 0] and s.attrs["tiles"] == 0.25 and s.attrs["randoms.W"] == 100.
    np.testing.assert_array_equal(s.attrs["BoxCenter"], [1., 2., 3.])
