"""
TEST INFRASTRUCTURE -- CPU restatement of the pair-count contract of nbodykit_b200/algorithms/paircount.py (DESIGN.md
4.6).

Positions are used as stored; periodic: wrapped with numpy's `pos % L` in their own dtype.  Columns are reordered so
that the line of sight c is last (a < b the other two axes).  Per axis |d| in float64 (periodic: min(|d|, L - |d|)),
r_p^2 = da^2 + db^2, s^2 = r_p^2 + dc^2.  Bin k of `edges` holds e_k^2 <= x^2 < e_{k+1}^2 (x = s, or r_p in
'projected'); '2d': mu = |dc| / s over linspace(0, 1, Nmu + 1), right-open, mu = 1 in the last bin; 'projected': only
|dc| < pimax, pi bins over linspace(0, pimax, int(pimax + 1)), right-open.  Pairs are ordered: (i, j) and (j, i) both
count in an auto count.  Candidates come from scipy's cKDTree at a radius above s_max, then this exact rule decides.
"""
import numpy as np


def second_edges(mode, Nmu=None, pimax=None):
    if mode == "2d":
        return np.linspace(0., 1., Nmu + 1)
    if mode == "projected":
        return np.linspace(0, pimax, int(pimax + 1))
    return None


def _prepare(pos, box, los):
    pos = np.asarray(pos)
    if box is not None:
        pos = np.mod(pos, np.asarray(box).astype(pos.dtype))
    axes = [i for i in range(3) if i != los] + [los]
    return pos[:, axes].astype("f8"), (np.asarray(box, "f8")[axes] if box is not None else None)


def _bin_pairs(a, b, w1, w2, mode, edges, box, Nmu, pimax):
    """(flat bin index, w1 * w2, separation) of the pairs of rows a[k], b[k] that count"""
    d = np.abs(a - b)
    if box is not None:
        d = np.minimum(d, box - d)
    rp2 = d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]
    e2 = np.asarray(edges, "f8") ** 2
    nb = len(e2) - 1
    if mode == "projected":
        x2 = rp2
        keep = (d[:, 2] < pimax) & (x2 >= e2[0]) & (x2 < e2[-1])
    else:
        x2 = rp2 + d[:, 2] * d[:, 2]
        keep = (x2 >= e2[0]) & (x2 < e2[-1])
    x2, dc = x2[keep], d[keep, 2]
    k = np.searchsorted(e2, x2, side="right") - 1
    sep = np.sqrt(x2)
    if mode == "1d":
        idx = k
    else:
        e = second_edges(mode, Nmu, pimax)
        n2 = len(e) - 1
        v = dc / sep if mode == "2d" else dc
        j = np.clip(np.searchsorted(e, v, side="right") - 1, 0, n2 - 1)
        idx = k * n2 + j
    return idx, w1[keep] * w2[keep], sep, nb


def _histogram(parts, mode, edges, Nmu, pimax):
    nb = len(edges) - 1
    e = second_edges(mode, Nmu, pimax)
    shape = (nb,) if e is None else (nb, len(e) - 1)
    nbins = int(np.prod(shape))
    npairs = np.zeros(nbins, "u8")
    # the per-pair terms are float64; their sums are taken in extended precision, so that the oracle's own summation
    # order does not use up the tolerance of the comparison
    wsum = np.zeros(nbins, np.longdouble)
    ssum = np.zeros(nbins, np.longdouble)
    for idx, ww, sep, _ in parts:
        npairs += np.bincount(idx, minlength=nbins).astype("u8")
        np.add.at(wsum, idx, ww.astype(np.longdouble))
        np.add.at(ssum, idx, sep.astype(np.longdouble))
    return dict(npairs=npairs.reshape(shape), wnpairs=wsum.astype("f8").reshape(shape),
                sepsum=ssum.astype("f8").reshape(shape))


def _smax(mode, edges, pimax):
    e = float(np.max(edges))
    return np.sqrt(e * e + pimax * pimax) if mode == "projected" else e


def count(pos1, mode, edges, box=None, pos2=None, w1=None, w2=None, los=2, Nmu=None, pimax=None, chunk=200000):
    """dict(npairs u8, wnpairs f8, sepsum f8) shaped like the result; box None: not periodic"""
    from scipy.spatial import cKDTree
    auto = pos2 is None
    a, boxr = _prepare(pos1, box, los)
    b, _ = _prepare(pos1 if auto else pos2, box, los)
    w1 = np.ones(len(a)) if w1 is None else np.asarray(w1, "f8")
    w2 = (w1 if auto else np.ones(len(b))) if w2 is None else np.asarray(w2, "f8")
    smax = _smax(mode, edges, pimax)
    if boxr is not None:
        # the tree needs [0, L): L_f4 may round above L_f8, so query with a margin over that shift as well
        t1 = cKDTree(np.mod(a, boxr), boxsize=boxr)
        t2 = cKDTree(np.mod(b, boxr), boxsize=boxr)
        r = smax * (1 + 1e-9) + 4e-7 * float(boxr.max())
    else:
        t1, t2 = cKDTree(a), cKDTree(b)
        r = smax * (1 + 1e-9)
    m = t1.sparse_distance_matrix(t2, r, output_type="ndarray")
    parts = []
    for s in range(0, len(m), chunk):
        i, j = m["i"][s:s + chunk], m["j"][s:s + chunk]
        parts.append(_bin_pairs(a[i], b[j], w1[i], w2[j], mode, edges, boxr, Nmu, pimax))
    # pairs at distance 0 never count (edges > 0), whether or not the tree lists them
    return _histogram(parts, mode, edges, Nmu, pimax)


def brute_force(pos1, mode, edges, box=None, pos2=None, w1=None, w2=None, los=2, Nmu=None, pimax=None):
    """the same contract over all N1 x N2 ordered pairs (small N only)"""
    auto = pos2 is None
    a, boxr = _prepare(pos1, box, los)
    b, _ = _prepare(pos1 if auto else pos2, box, los)
    w1 = np.ones(len(a)) if w1 is None else np.asarray(w1, "f8")
    w2 = (w1 if auto else np.ones(len(b))) if w2 is None else np.asarray(w2, "f8")
    i, j = np.meshgrid(np.arange(len(a)), np.arange(len(b)), indexing="ij")
    i, j = i.ravel(), j.ravel()
    return _histogram([_bin_pairs(a[i], b[j], w1[i], w2[j], mode, edges, boxr, Nmu, pimax)], mode, edges, Nmu, pimax)


def clustered(seed, L, n_bg, blobs, size, scale, dtype="f8"):
    """uniform background plus `blobs` gaussian blobs of `size` rows each, wrapped into [0, L)"""
    rng = np.random.RandomState(seed)
    parts = [rng.uniform(size=(n_bg, 3)) * L]
    for _ in range(blobs):
        parts.append(rng.uniform(size=3) * L + rng.normal(scale=scale, size=(size, 3)))
    return np.mod(np.concatenate(parts), L).astype(dtype)
