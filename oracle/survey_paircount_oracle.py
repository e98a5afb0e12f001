"""
TEST INFRASTRUCTURE -- CPU restatement of the survey pair-count contract of
nbodykit_b200/algorithms/surveypaircount.py (DESIGN.md 4.8).

Rows are Cartesian float64 positions with the observer at the origin ('angular': unit vectors), used as given.  For a
primary x1 and a secondary x2, per axis s = x2 - x1 and l = x1 + x2; s^2 = (sx^2 + sy^2) + sz^2,
l^2 = (lx^2 + ly^2) + lz^2, sl = (sx lx + sy ly) + sz lz, all in float64 with no FMA.  Bin k of `edges` holds
e_k^2 <= x^2 < e_{k+1}^2.
  '1d'        : x = s, summing s.
  '2d'        : x = s, mu = |sl| / (sqrt(s^2) sqrt(l^2)) (0 when l^2 = 0) over linspace(0, 1, Nmu + 1), right-open,
                mu >= 1 in the last bin; summing s.
  'projected' : pi = |sl| / sqrt(l^2) (0 when l^2 = 0), only pi < pimax; r_p^2 = max(s^2 - pi pi, 0) is x^2, pi bins
                over linspace(0, pimax, int(pimax + 1)), right-open; summing r_p.
  'angular'   : the edges are theta in degrees, binned as chords c = 2 sin(theta / 2); x^2 = s^2; summing
                theta = 2 asin(0.5 sqrt(s^2)) (180 / pi).
Pairs are ordered: (i, j) and (j, i) both count in an auto count.  Candidates come from scipy's cKDTree at a radius
above the largest separation that can count, then this exact rule decides; `brute_force` applies it to every pair.
"""
import numpy as np


def second_edges(mode, Nmu=None, pimax=None):
    if mode == "2d":
        return np.linspace(0., 1., Nmu + 1)
    if mode == "projected":
        return np.linspace(0, pimax, int(pimax + 1))
    return None


def chord_edges(theta):
    return 2. * np.sin(0.5 * np.deg2rad(np.asarray(theta, dtype="f8")))


def _kernel_edges(mode, edges):
    return chord_edges(edges) if mode == "angular" else np.asarray(edges, "f8")


def _bin_pairs(a, b, w1, w2, mode, edges, Nmu, pimax):
    """(flat bin index, w1 * w2, summed separation) of the pairs of rows a[k] (primary), b[k] (secondary) that count"""
    s = b - a
    ell = a + b
    s2 = (s[:, 0] * s[:, 0] + s[:, 1] * s[:, 1]) + s[:, 2] * s[:, 2]
    e2 = _kernel_edges(mode, edges) ** 2
    if mode == "projected":
        l2 = (ell[:, 0] * ell[:, 0] + ell[:, 1] * ell[:, 1]) + ell[:, 2] * ell[:, 2]
        sl = (s[:, 0] * ell[:, 0] + s[:, 1] * ell[:, 1]) + s[:, 2] * ell[:, 2]
        with np.errstate(invalid="ignore", divide="ignore"):
            pi = np.where(l2 > 0, np.abs(sl) / np.sqrt(l2), 0.)
        x2 = np.maximum(s2 - pi * pi, 0.)
        keep = (pi < pimax) & (x2 >= e2[0]) & (x2 < e2[-1])
    else:
        x2 = s2
        keep = (x2 >= e2[0]) & (x2 < e2[-1])
    x2 = x2[keep]
    k = np.searchsorted(e2, x2, side="right") - 1
    if mode == "angular":
        sep = 2. * np.arcsin(0.5 * np.sqrt(x2)) * (180. / np.pi)
    else:
        sep = np.sqrt(x2)
    if mode in ("1d", "angular"):
        return k, w1[keep] * w2[keep], sep
    e = second_edges(mode, Nmu, pimax)
    n2 = len(e) - 1
    if mode == "2d":
        sk, lk = s[keep], ell[keep]
        l2 = (lk[:, 0] * lk[:, 0] + lk[:, 1] * lk[:, 1]) + lk[:, 2] * lk[:, 2]
        sl = (sk[:, 0] * lk[:, 0] + sk[:, 1] * lk[:, 1]) + sk[:, 2] * lk[:, 2]
        with np.errstate(invalid="ignore", divide="ignore"):
            v = np.where(l2 > 0, np.abs(sl) / (sep * np.sqrt(l2)), 0.)
    else:
        v = pi[keep]
    j = np.clip(np.searchsorted(e, v, side="right") - 1, 0, n2 - 1)
    return k * n2 + j, w1[keep] * w2[keep], sep


def _histogram(parts, mode, edges, Nmu, pimax):
    nb = len(edges) - 1
    e = second_edges(mode, Nmu, pimax)
    shape = (nb,) if e is None else (nb, len(e) - 1)
    nbins = int(np.prod(shape))
    npairs = np.zeros(nbins, "u8")
    # float64 per-pair terms, summed in extended precision (as oracle/paircount_oracle.py)
    wsum = np.zeros(nbins, np.longdouble)
    ssum = np.zeros(nbins, np.longdouble)
    for idx, ww, sep in parts:
        npairs += np.bincount(idx, minlength=nbins).astype("u8")
        np.add.at(wsum, idx, ww.astype(np.longdouble))
        np.add.at(ssum, idx, sep.astype(np.longdouble))
    return dict(npairs=npairs.reshape(shape), wnpairs=wsum.astype("f8").reshape(shape),
                sepsum=ssum.astype("f8").reshape(shape))


def _prepare(pos1, pos2, w1, w2):
    a = np.asarray(pos1, "f8")
    b = a if pos2 is None else np.asarray(pos2, "f8")
    w1 = np.ones(len(a)) if w1 is None else np.asarray(w1, "f8")
    w2 = (w1 if pos2 is None else np.ones(len(b))) if w2 is None else np.asarray(w2, "f8")
    return a, b, w1, w2


def count(pos1, mode, edges, pos2=None, w1=None, w2=None, Nmu=None, pimax=None, chunk=200000):
    """dict(npairs u8, wnpairs f8, sepsum f8) shaped like the result"""
    from scipy.spatial import cKDTree
    a, b, w1, w2 = _prepare(pos1, pos2, w1, w2)
    e = _kernel_edges(mode, edges)
    smax = float(e[-1])
    if mode == "projected":
        smax = np.sqrt(smax * smax + pimax * pimax)
    m = cKDTree(a).sparse_distance_matrix(cKDTree(b), smax * (1 + 1e-9), output_type="ndarray")
    parts = []
    for s in range(0, len(m), chunk):
        i, j = m["i"][s:s + chunk], m["j"][s:s + chunk]
        parts.append(_bin_pairs(a[i], b[j], w1[i], w2[j], mode, edges, Nmu, pimax))
    # pairs at distance 0 never count (edges > 0), whether or not the tree lists them
    return _histogram(parts, mode, edges, Nmu, pimax)


def brute_force(pos1, mode, edges, pos2=None, w1=None, w2=None, Nmu=None, pimax=None):
    """the same contract over all N1 x N2 ordered pairs (small N only)"""
    a, b, w1, w2 = _prepare(pos1, pos2, w1, w2)
    i, j = np.meshgrid(np.arange(len(a)), np.arange(len(b)), indexing="ij")
    i, j = i.ravel(), j.ravel()
    return _histogram([_bin_pairs(a[i], b[j], w1[i], w2[j], mode, edges, Nmu, pimax)], mode, edges, Nmu, pimax)


def sky_catalogue(seed, n, ra=(110., 260.), dec=(-3.6, 60.), z=(0.5, 0.1)):
    """(RA, Dec, z) uniform in RA and Dec over the given ranges, z normal with (mean, sigma) and kept above 0.01"""
    rng = np.random.RandomState(seed)
    r = rng.uniform(ra[0], ra[1], n)
    d = rng.uniform(dec[0], dec[1], n)
    zz = np.abs(rng.normal(z[0], z[1], n)) + 0.01
    return r, d, zz
