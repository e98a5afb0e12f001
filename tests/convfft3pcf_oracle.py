"""Float64 NumPy oracle of ConvolvedFFT3PCF (DESIGN.md §4.17).  N and Rf are real fields on the full mesh (shape Nmesh)
that are zero wherever a pair within max(edges) could wrap (the class's geometry guard); separations are true grid
separations s = n H, r = sqrt((sx^2 + sy^2) + sz^2), bin b holding e_b < r <= e_{b+1} and r > 0;

    nnn_l(b1, b2) = (2l + 1) / (16 pi^2) sum_x N(x) sum_{s1 in b1} sum_{s2 in b2} N(x + s1) N(x + s2) P_l(u1.u2)

and rrr_l the same with Rf.  No mean is subtracted.

Two independent forms:
  fft_form    -- the method with scipy's real Y_lm and numpy.fft on the periodic mesh, as fft3pcf_oracle.fft_form but
                 without the mean: a_lm,b = irfftn(rfftn(W) conj(rfftn(Y_lm 1_b))), sum = (1 / 4 pi) sum_m sum_x W a a;
  direct_form -- every cell and every true separation enumerated, no wrap (a shift that leaves the mesh reads 0), with
                 T(s1, s2) = sum_x W(x) W(x + s1) W(x + s2) as one matrix product weighted by the Legendre polynomial of
                 u1.u2 (no Y_lm, no FFT).  Meshes of at most 12^3 cells.
bound_l = (2l + 1) / (16 pi^2) sum_x |W| (sum_{s1} |W|) (sum_{s2} |W|) bounds |nnn_l| (W = N) and |rrr_l| (W = Rf) and
scales the tolerances."""
import numpy as np
from scipy.special import eval_legendre

import fft3pcf_oracle as fo


def _conv(f, K):
    return np.fft.irfftn(np.fft.rfftn(f) * np.conj(np.fft.rfftn(K)), s=f.shape, axes=(0, 1, 2))


def _bound(W, b, nb, poles):
    a = np.abs(np.asarray(W, dtype="f8"))
    c = [_conv(a, (b == k).astype("f8")) for k in range(nb)]
    base = np.array([[np.sum(a * c[i] * c[j]) for j in range(nb)] for i in range(nb)])
    return np.array([(2 * ell + 1) / (16 * np.pi ** 2) * base for ell in poles])


def _fft_sum(W, Nmesh, BoxSize, edges, poles):
    W = np.asarray(W, dtype="f8")
    sx, sy, sz, r = fo.separations(Nmesh, BoxSize)
    b = fo.bins(Nmesh, BoxSize, edges)
    nb = len(edges) - 1
    wh = np.fft.rfftn(W)
    out = np.zeros((len(poles), nb, nb))
    for p, ell in enumerate(poles):
        for m in range(-ell, ell + 1):
            Y = fo.real_ylm(ell, m, sx, sy, sz, r)
            a = [np.fft.irfftn(wh * np.conj(np.fft.rfftn(np.where(b == k, Y, 0.0))), s=W.shape, axes=(0, 1, 2))
                 for k in range(nb)]
            for i in range(nb):
                wa = W * a[i]
                for j in range(nb):
                    out[p, i, j] += np.sum(wa * a[j])
        out[p] /= 4 * np.pi
    return out


def _direct_sum(W, Nmesh, BoxSize, edges, poles):
    W = np.asarray(W, dtype="f8")
    N = W.shape
    sx, sy, sz, r = fo.separations(Nmesh, BoxSize)
    b = fo.bins(Nmesh, BoxSize, edges)
    nb = len(edges) - 1
    idx = np.argwhere(b >= 0)                                    # cell offsets of the separations in a bin
    which = b[tuple(idx.T)]
    n = np.stack([np.where(2 * idx[:, d] <= N[d], idx[:, d], idx[:, d] - N[d]) for d in range(3)], axis=1)
    u = np.stack([sx[tuple(idx.T)], sy[tuple(idx.T)], sz[tuple(idx.T)]], axis=1) / r[tuple(idx.T)][:, None]
    x = np.indices(N).reshape(3, -1)
    D = np.zeros((len(idx), x.shape[1]))
    for q, o in enumerate(n):
        y = x + o[:, None]
        inside = ((y >= 0) & (y < np.array(N)[:, None])).all(axis=0)
        D[q, inside] = W[y[0, inside], y[1, inside], y[2, inside]]
    T = (D * W.reshape(-1)[None, :]) @ D.T
    mu = np.clip(u @ u.T, -1, 1)
    sel = np.stack([which == k for k in range(nb)]).astype("f8")
    out = np.zeros((len(poles), nb, nb))
    for p, ell in enumerate(poles):
        out[p] = (2 * ell + 1) / (16 * np.pi ** 2) * (sel @ (T * eval_legendre(ell, mu)) @ sel.T)
    return out


def _form(sum_, N, Rf, Nmesh, BoxSize, edges, poles):
    b = fo.bins(Nmesh, BoxSize, edges)
    nb = len(edges) - 1
    return dict(nnn=sum_(N, Nmesh, BoxSize, edges, poles), rrr=sum_(Rf, Nmesh, BoxSize, edges, poles),
                nsep=fo.nsep(Nmesh, BoxSize, edges), bound_n=_bound(N, b, nb, poles), bound_r=_bound(Rf, b, nb, poles))


def fft_form(N, Rf, Nmesh, BoxSize, edges, poles):
    """dict(nnn, rrr, bound_n, bound_r: (npoles, nb, nb); nsep) by the addition theorem"""
    return _form(_fft_sum, N, Rf, Nmesh, BoxSize, edges, poles)


def direct_form(N, Rf, Nmesh, BoxSize, edges, poles):
    """dict(nnn, rrr, bound_n, bound_r; nsep) from every cell and every true separation"""
    return _form(_direct_sum, N, Rf, Nmesh, BoxSize, edges, poles)
