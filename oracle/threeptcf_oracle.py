"""
TEST INFRASTRUCTURE -- CPU restatement of the three-point contract of nbodykit_b200/algorithms/threeptcf.py (DESIGN.md
4.7).

Positions are used as stored; periodic: wrapped with numpy's `pos % L` in their own dtype, then widened to float64.
For a primary p and a secondary j, d = x_j - x_p per axis in float64 (periodic: d > L/2 -> d - L, d <= -L/2 -> d + L),
r = sqrt((dx^2 + dy^2) + dz^2); j is in radial bin k when e_k < r <= e_{k+1} (searchsorted side='left'), and r > 0.

    zeta_l(b1, b2) = (2l + 1) / (16 pi^2) sum_p w_p sum_{j in b1} sum_{k in b2} w_j w_k P_l(u_pj . u_pk)
                   = 1 / (4 pi) sum_p w_p sum_{m=-l}^{l} Re[a_lm(b1) a*_lm(b2)],   a_lm(b) = sum_{j in b} w_j Y_lm(u_pj)

compute() takes the neighbours from scipy's cKDTree at a radius above r_max and applies these rules exactly, forming
a_lm with scipy.special.sph_harm_y; brute_force() evaluates the Legendre form over all pairs (small N).  Both return
dict(zeta [npoles][nb][nb], npairs u8 [nb], bound [npoles][nb][nb]) with the bound
B_l(b1, b2) = (2l + 1) / (16 pi^2) sum_p |w_p| S_p(b1) S_p(b2), S_p(b) = sum_{j in b} |w_j|, so that |zeta_l| <= B_l.
"""
import numpy as np


def _prepare(pos, box):
    pos = np.asarray(pos)
    if box is not None:
        pos = np.mod(pos, np.asarray(box).astype(pos.dtype))
    return pos.astype("f8"), (np.asarray(box, "f8") * np.ones(3) if box is not None else None)


def _pairs_binned(a, i, j, edges, box):
    """(i, j, bin, d, r) of the ordered pairs (primary a[i], secondary a[j]) that count"""
    d = a[j] - a[i]
    if box is not None:
        h = 0.5 * box
        d = np.where(d > h, d - box, np.where(d <= -h, d + box, d))
    r = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    e = np.asarray(edges, "f8")
    k = np.searchsorted(e, r, side="left") - 1
    keep = (r > 0) & (k >= 0) & (k < len(e) - 1)
    return i[keep], j[keep], k[keep], d[keep], r[keep]


def _bound(w, i, j, k, n, nb, poles):
    S = np.bincount(i * nb + k, weights=np.abs(w[j]), minlength=n * nb).reshape(n, nb)
    SS = np.einsum("p,pa,pb->ab", np.abs(w), S, S)
    return np.array([(2 * ell + 1) / (16 * np.pi ** 2) * SS for ell in poles])


def neighbours(pos, edges, box=None):
    """(primary index, secondary index, bin, d, r) of every ordered pair that counts, from cKDTree candidates"""
    from scipy.spatial import cKDTree
    a, boxr = _prepare(pos, box)
    rmax = float(np.max(edges))
    if boxr is not None:
        # the tree needs [0, L): L_f4 may round above L_f8, so query with a margin over that shift as well
        t = cKDTree(np.mod(a, boxr), boxsize=boxr)
        rq = rmax * (1 + 1e-9) + 4e-7 * float(boxr.max())
    else:
        t = cKDTree(a)
        rq = rmax * (1 + 1e-9)
    m = t.sparse_distance_matrix(t, rq, output_type="ndarray")
    # pairs at distance 0 (self pairs, duplicates) never count, whether or not the tree lists them
    return _pairs_binned(a, m["i"].astype(np.int64), m["j"].astype(np.int64), edges, boxr)


def compute(pos, edges, poles, box=None, w=None, chunk=2000000):
    """the contract through a_lm = sum_j w_j Y_lm(u_pj) (scipy.special.sph_harm_y); box None: not periodic"""
    from scipy.special import sph_harm_y
    a, _ = _prepare(pos, box)
    n = len(a)
    w = np.ones(n) if w is None else np.asarray(w, "f8")
    nb = len(edges) - 1
    i, j, k, d, r = neighbours(pos, edges, box)
    order = np.argsort(i, kind="stable")
    i, j, k, d, r = i[order], j[order], k[order], d[order], r[order]
    theta = np.arccos(np.clip(d[:, 2] / r, -1., 1.))
    phi = np.arctan2(d[:, 1], d[:, 0])
    wj = w[j]
    idx = i * nb + k
    zeta = np.zeros((len(poles), nb, nb))
    for ip, ell in enumerate(poles):
        for m in range(ell + 1):
            alm = np.zeros(n * nb, complex)
            for s in range(0, len(i), chunk):
                y = wj[s:s + chunk] * sph_harm_y(ell, m, theta[s:s + chunk], phi[s:s + chunk])
                alm += np.bincount(idx[s:s + chunk], weights=y.real, minlength=n * nb)
                alm += 1j * np.bincount(idx[s:s + chunk], weights=y.imag, minlength=n * nb)
            alm = alm.reshape(n, nb)
            t = np.einsum("p,pa,pb->ab", w, alm, alm.conj()).real
            zeta[ip] += (1. if m == 0 else 2.) * t
    zeta /= 4 * np.pi
    npairs = np.bincount(k, minlength=nb).astype("u8")
    return dict(zeta=zeta, npairs=npairs, bound=_bound(w, i, j, k, n, nb, poles))


def brute_force(pos, edges, poles, box=None, w=None):
    """the Legendre form of the contract over all N x N ordered pairs (small N only)"""
    from scipy.special import eval_legendre
    a, boxr = _prepare(pos, box)
    n = len(a)
    w = np.ones(n) if w is None else np.asarray(w, "f8")
    nb = len(edges) - 1
    ii, jj = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    i, j, k, d, r = _pairs_binned(a, ii.ravel(), jj.ravel(), edges, boxr)
    zeta = np.zeros((len(poles), nb, nb))
    for p in np.unique(i):
        sel = i == p
        u = d[sel] / r[sel][:, None]
        c = np.clip(u @ u.T, -1., 1.)
        B = np.zeros((sel.sum(), nb))
        B[np.arange(sel.sum()), k[sel]] = w[j[sel]]
        for ip, ell in enumerate(poles):
            zeta[ip] += w[p] * (B.T @ eval_legendre(ell, c) @ B)
    for ip, ell in enumerate(poles):
        zeta[ip] *= (2 * ell + 1) / (16 * np.pi ** 2)
    npairs = np.bincount(k, minlength=nb).astype("u8")
    return dict(zeta=zeta, npairs=npairs, bound=_bound(w, i, j, k, n, nb, poles))


def golden():
    """(positions, weights, truth[8][8][11]) of the reference's test data: 1000 weighted points in L = 400, and the
    result of Daniel Eisenstein's C++ code for 8 bins over [0, 200] and l = 0 .. 10, normalised as
    zeta_l (4 pi)^2 / (2l + 1)"""
    import os
    here = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
    d = np.loadtxt(os.path.join(here, "threeptcf_sim_data.dat"))
    truth = np.empty((8, 8, 11))
    with open(os.path.join(here, "threeptcf_sim_result.dat")) as ff:
        for line in ff:
            f = line.split()
            p, q = int(f[0]), int(f[1])
            truth[p, q] = list(map(float, f[2:]))
            truth[q, p] = truth[p, q]
    return d[:, :3] * 400., d[:, 3], truth


def clustered(seed, L, n_bg, blobs, size, scale, dtype="f8"):
    """uniform background plus `blobs` gaussian blobs of `size` rows each, wrapped into [0, L)"""
    rng = np.random.RandomState(seed)
    parts = [rng.uniform(size=(n_bg, 3)) * L]
    for _ in range(blobs):
        parts.append(rng.uniform(size=3) * L + rng.normal(scale=scale, size=(size, 3)))
    return np.mod(np.concatenate(parts), L).astype(dtype)
