"""Float64 NumPy oracle of FFT3PCF (DESIGN.md §4.16).  F is a real field on the full mesh (shape Nmesh), delta = F -
mean(F); grid separations s = n H with n_i in (-N_i/2, N_i/2] and H_i = L_i / N_i; r = sqrt((sx^2 + sy^2) + sz^2);
bin b holds e_b < r <= e_{b+1} and r > 0;

    corr_l(b1, b2) = (2l + 1) / (16 pi^2) sum_x delta(x) sum_{s1 in b1} sum_{s2 in b2} delta(x + s1) delta(x + s2) P_l(u1.u2)
    zeta_l(b1, b2) = 16 pi^2 corr_l / (N_cells nsep[b1] nsep[b2])

Two independent forms:
  fft_form    -- the addition theorem with scipy's Y_lm, real orthonormal: a_lm,b = irfftn(rfftn(delta)
                 conj(rfftn(Y_lm 1_b))) = sum_{s in b} Y_lm(u) delta(x + s), corr_l = (1 / 4 pi) sum_m sum_x delta a a;
  direct_form -- every separation of every bin enumerated: T(s1, s2) = sum_x delta(x) delta(x + s1) delta(x + s2) as one
                 matrix product, weighted by the Legendre polynomial of u1.u2 (no Y_lm, no FFT).  Small meshes only.
bound_l = (2l + 1) / (16 pi^2) sum_x |delta| (sum_{s1} |delta|) (sum_{s2} |delta|) bounds |corr_l| and scales the
tolerances."""
import numpy as np
from scipy.special import eval_legendre, sph_harm_y


def separations(Nmesh, BoxSize):
    """(sx, sy, sz, r) on the full mesh, indexed by the cell offset of the separation"""
    N = [int(v) for v in np.broadcast_to(Nmesh, 3)]
    L = np.broadcast_to(np.asarray(BoxSize, dtype="f8"), 3)
    s = []
    for d in range(3):
        i = np.arange(N[d])
        n = np.where(2 * i <= N[d], i, i - N[d]).astype("f8")
        shape = [1, 1, 1]
        shape[d] = N[d]
        s.append(np.broadcast_to((n * (L[d] / N[d])).reshape(shape), N))
    sx, sy, sz = s
    r = np.sqrt((sx * sx + sy * sy) + sz * sz)
    return sx, sy, sz, r


def bins(Nmesh, BoxSize, edges):
    """the radial bin of every separation (-1: in none)"""
    e = np.asarray(edges, dtype="f8")
    r = separations(Nmesh, BoxSize)[3]
    b = np.full(r.shape, -1, dtype="i8")
    for k in range(len(e) - 1):
        b[(r > 0) & (r > e[k]) & (r <= e[k + 1])] = k
    return b


def nsep(Nmesh, BoxSize, edges):
    b = bins(Nmesh, BoxSize, edges)
    return np.array([(b == k).sum() for k in range(len(edges) - 1)], dtype="u8")


def real_ylm(ell, m, sx, sy, sz, r):
    """real orthonormal Y_lm(s / r): m = 0 Y_l0, m > 0 sqrt(2) Re Y_lm, m < 0 sqrt(2) Im Y_l|m| (0 where r = 0)"""
    with np.errstate(invalid="ignore", divide="ignore"):
        theta = np.arccos(np.clip(np.where(r > 0, sz / r, 1.0), -1, 1))
    phi = np.arctan2(sy, sx)
    y = sph_harm_y(ell, abs(m), theta, phi)
    if m == 0:
        return y.real
    return np.sqrt(2.) * (y.real if m > 0 else y.imag)


def _delta(F):
    F = np.asarray(F, dtype="f8")
    return F - F.sum() / F.size


def _conv(f, K):
    """sum_s K(s) f(x + s) on the periodic mesh"""
    return np.fft.irfftn(np.fft.rfftn(f) * np.conj(np.fft.rfftn(K)), s=f.shape, axes=(0, 1, 2))


def bound(F, Nmesh, BoxSize, edges, poles):
    """(npoles, nb, nb) bound_l"""
    d = np.abs(_delta(F))
    b = bins(Nmesh, BoxSize, edges)
    nb = len(edges) - 1
    c = [_conv(d, (b == k).astype("f8")) for k in range(nb)]
    base = np.array([[np.sum(d * c[i] * c[j]) for j in range(nb)] for i in range(nb)])
    return np.array([(2 * ell + 1) / (16 * np.pi ** 2) * base for ell in poles])


def _finish(corr, ns, ncell):
    with np.errstate(invalid="ignore", divide="ignore"):
        nn = np.outer(ns.astype("f8"), ns.astype("f8"))
        zeta = np.where(nn > 0, 16 * np.pi ** 2 * corr / (ncell * nn), np.nan)
    return zeta


def fft_form(F, Nmesh, BoxSize, edges, poles):
    """dict(corr, zeta, bound: (npoles, nb, nb); nsep: (nb,) u8) by the addition theorem"""
    d = _delta(F)
    sx, sy, sz, r = separations(Nmesh, BoxSize)
    b = bins(Nmesh, BoxSize, edges)
    nb = len(edges) - 1
    dh = np.fft.rfftn(d)
    corr = np.zeros((len(poles), nb, nb))
    for p, ell in enumerate(poles):
        for m in range(-ell, ell + 1):
            Y = real_ylm(ell, m, sx, sy, sz, r)
            a = [np.fft.irfftn(dh * np.conj(np.fft.rfftn(np.where(b == k, Y, 0.0))), s=d.shape, axes=(0, 1, 2)) for k in range(nb)]
            for i in range(nb):
                da = d * a[i]
                for j in range(nb):
                    corr[p, i, j] += np.sum(da * a[j])
        corr[p] /= 4 * np.pi
    ns = np.array([(b == k).sum() for k in range(nb)], dtype="u8")
    return dict(corr=corr, zeta=_finish(corr, ns, d.size), nsep=ns, bound=bound(F, Nmesh, BoxSize, edges, poles))


def direct_form(F, Nmesh, BoxSize, edges, poles):
    """dict(corr, zeta: (npoles, nb, nb); nsep) from every pair of separations, with explicit Legendre polynomials"""
    d = _delta(F)
    N = d.shape
    sx, sy, sz, r = separations(Nmesh, BoxSize)
    b = bins(Nmesh, BoxSize, edges)
    nb = len(edges) - 1
    idx = np.argwhere(b >= 0)                                   # (nsep_total, 3) cell offsets
    which = b[tuple(idx.T)]
    u = np.stack([sx[tuple(idx.T)], sy[tuple(idx.T)], sz[tuple(idx.T)]], axis=1) / r[tuple(idx.T)][:, None]
    # D[q, x] = delta(x + s_q): every cell enumerated for every separation
    x = np.indices(N).reshape(3, -1)
    D = np.empty((len(idx), x.shape[1]))
    for q, o in enumerate(idx):
        D[q] = d[(x[0] + o[0]) % N[0], (x[1] + o[1]) % N[1], (x[2] + o[2]) % N[2]]
    T = (D * d.reshape(-1)[None, :]) @ D.T                     # sum_x delta(x) delta(x + s1) delta(x + s2)
    mu = np.clip(u @ u.T, -1, 1)
    sel = np.stack([which == k for k in range(nb)]).astype("f8")   # (nb, nsep_total)
    corr = np.zeros((len(poles), nb, nb))
    for p, ell in enumerate(poles):
        corr[p] = (2 * ell + 1) / (16 * np.pi ** 2) * (sel @ (T * eval_legendre(ell, mu)) @ sel.T)
    ns = np.array([(which == k).sum() for k in range(nb)], dtype="u8")
    return dict(corr=corr, zeta=_finish(corr, ns, d.size), nsep=ns)
