"""
TEST INFRASTRUCTURE -- float64 NumPy oracle for the multipoles of FFTBispectrum (poles=, los=; DESIGN.md 4.14).
NOT product code.  Shells, triples and the full-grid spectrum are those of oracle/bispectrum_oracle.py.

mu = q.los / |q| is formed in float32 as FFTPower forms it for a Python-number los: k from pmesh_oracle.k_coords
(coord_dtype="f4"), ((kx l0 + ky l1) + kz l2) / sqrt(k2) with k2 = (kx^2 + ky^2) + kz^2, then L_ell(mu) in float64 by
the recurrence of the binning kernel.  The weight sits on the first wavevector (shell a); rows are (a, b, c), b <= c.

  fft_form_poles    -- W^ell_a = c2r(c L_ell 1_Sa), I, J as in fft_form; B_ell = (2 ell + 1) V^2 sum W_a I_b I_c / sum J J J
                       and bound_ell = (2 ell + 1) V^2 sum |W_a||I_b||I_c| / sum J J J per row
  direct_form_poles -- no FFT: sum over q1 in S_a, q2 in S_b with q3 = -(q1 + q2) modulo the grid in S_c of
                       L_ell(mu(q1)) c(q1) c(q2) c(q3)
"""
import numpy as np

from oracle import bispectrum_oracle as bo
from oracle import pmesh_oracle as po


def legendre(ell, x):
    """L_ell(x) in float64, the recurrence of the binning kernel"""
    x = np.asarray(x, dtype="f8")
    if ell == 0:
        return np.ones_like(x)
    p0, p1 = np.ones_like(x), x
    for n in range(1, ell):
        p0, p1 = p1, ((2 * n + 1) * x * p1 - n * p0) / (n + 1)
    return p1


def pole_rows(kedges):
    """(a, b, c), b <= c, for every distinct shell a of every evaluated sorted triple, in triple order"""
    rows = []
    for i, j, l in bo.triples(kedges).tolist():
        for a in sorted({i, j, l}):
            rest = [i, j, l]
            rest.remove(a)
            rows.append([a] + rest)
    return np.array(rows, dtype="i8").reshape(-1, 3)


def _mu(kx, ky, kz, los):
    """mu at float32 coordinates, in float32 (0 at k = 0)"""
    l0, l1, l2 = [np.float32(v) for v in los]
    k2 = (kx * kx + ky * ky) + kz * kz
    lp = kx * l0 + ky * l1
    with np.errstate(invalid="ignore", divide="ignore"):
        mu = (lp + kz * l2) / np.sqrt(k2)
    return np.where(k2 > 0, mu, np.float32(0)).astype("f4")


def mu_half(Nmesh, BoxSize, los):
    kx, ky, kz = po.k_coords(Nmesh, BoxSize, coord_dtype="f4")
    return _mu(kx, ky, kz, los)


def _setup(half, Nmesh, BoxSize):
    N = tuple(int(v) for v in np.asarray(Nmesh) * np.ones(3, dtype="i8"))
    L = np.asarray(BoxSize, dtype="f8") * np.ones(3)
    return N, L, float(np.prod(L)), float(np.prod(N)), np.asarray(half).astype("c16")


def fft_form_poles(half, Nmesh, BoxSize, kedges, poles, los):
    """{ell: dict(rows, S, B, bound, triangles, Tsum)} per row of pole_rows (ell = 0 included: the plain estimator)"""
    N, L, V, Nc, half = _setup(half, Nmesh, BoxSize)
    sh = bo.shells(N, L, kedges)
    n = len(kedges) - 1
    mu = mu_half(N, L, los).astype("f8")
    c2r = lambda a: np.fft.irfftn(a, s=N, axes=(0, 1, 2)) * Nc        # noqa: E731
    I = [c2r(np.where(sh == s, half, 0)) for s in range(n)]
    J = [c2r((sh == s).astype("c16")) for s in range(n)]
    rows = pole_rows(kedges)
    Tsum = np.array([np.sum(J[a] * J[b] * J[c]) for a, b, c in rows])
    count = np.rint(Tsum / Nc).astype("i8")
    out = {}
    for ell in poles:
        w = half * legendre(ell, mu)
        W = [c2r(np.where(sh == s, w, 0)) for s in range(n)]
        S = np.array([np.sum(W[a] * I[b] * I[c]) for a, b, c in rows])
        A = np.array([np.sum(np.abs(W[a] * I[b] * I[c])) for a, b, c in rows])
        with np.errstate(invalid="ignore", divide="ignore"):
            B = np.where(count > 0, (2 * ell + 1) * V ** 2 * S / Tsum, np.nan)
            bound = np.where(count > 0, (2 * ell + 1) * V ** 2 * A / Tsum, 0.)
        out[ell] = dict(rows=rows, S=S, B=B, bound=bound, triangles=count, Tsum=Tsum)
    return out


def direct_form_poles(half, Nmesh, BoxSize, kedges, poles, los):
    """{ell: dict(rows, B, triangles)} from a direct sum over closed triangles of the full grid (no FFT of the shells)"""
    N, L, V, Nc, half = _setup(half, Nmesh, BoxSize)
    c = np.fft.fftn(np.fft.irfftn(half, s=N, axes=(0, 1, 2)))
    sh = bo._full_shells(bo.shells(N, L, kedges), N)
    # float32 coordinates of the full grid: the mirror -q of a stored mode has mu(-q) = -mu(q) exactly
    k = [(np.fft.fftfreq(N[d]) * N[d]).round().astype("f4") * np.float32(2 * np.pi / L[d]) for d in range(3)]
    mu = _mu(k[0][:, None, None], k[1][None, :, None], k[2][None, None, :], los).astype("f8")
    n = len(kedges) - 1
    members = [np.argwhere(sh == s) for s in range(n)]
    Nv = np.array(N)
    S3, T3 = {}, {}
    for a in range(n):
        for b in range(n):
            q1, q2 = members[a], members[b]
            if len(q1) == 0 or len(q2) == 0:
                continue
            q3 = (-(q1[:, None, :] + q2[None, :, :])) % Nv
            s3 = sh[q3[..., 0], q3[..., 1], q3[..., 2]]
            val = (c[q1[:, 0], q1[:, 1], q1[:, 2]][:, None] * c[q2[:, 0], q2[:, 1], q2[:, 2]][None, :]
                   * c[q3[..., 0], q3[..., 1], q3[..., 2]])
            m1 = mu[q1[:, 0], q1[:, 1], q1[:, 2]][:, None] * np.ones(val.shape)
            ok = s3 >= 0
            T3[a, b] = np.bincount(s3[ok], minlength=n)
            for ell in poles:
                S3[ell, a, b] = np.bincount(s3[ok], weights=(legendre(ell, m1) * val)[ok].real, minlength=n)
    rows = pole_rows(kedges)
    count = np.array([T3[a, b][cc] if (a, b) in T3 else 0 for a, b, cc in rows], dtype="i8")
    out = {}
    for ell in poles:
        S = np.array([S3[ell, a, b][cc] if (ell, a, b) in S3 else 0. for a, b, cc in rows])
        with np.errstate(invalid="ignore", divide="ignore"):
            B = np.where(count > 0, (2 * ell + 1) * V ** 2 * S / count, np.nan)
        out[ell] = dict(rows=rows, B=B, triangles=count)
    return out
