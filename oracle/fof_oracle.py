"""
TEST INFRASTRUCTURE -- CPU restatement of the friends-of-friends contract (nbodykit_b200/algorithms/fof.py); pinned
against the reference's own helpers by tests/test_oracle_fof_reference.py (oracle/fof_refload.py).

Friends: d^2 = (dx^2 + dy^2) + dz^2 <= b^2 in float64 from the positions as stored; periodic: wrapped with numpy's
`pos % L` in their own dtype, per-axis |d| -> min(|d|, L - |d|).  Candidate pairs come from scipy's cKDTree (or brute
force for small n) and are then decided by that exact rule.  Groups are the connected components; labels 0 for N <= nmin,
else 1..H by (-N, minid); centres of mass are `centerofmass` (fof.py:647-700) in float64.
"""
import numpy as np


def wrapped(pos, box):
    pos = np.asarray(pos)
    return np.mod(pos, np.asarray(box).astype(pos.dtype))


def _d2(a, b, box):
    d = np.abs(a.astype("f8") - b.astype("f8"))
    if box is not None:
        d = np.minimum(d, np.asarray(box, "f8") - d)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def friend_pairs(pos, b, box=None, check_margin=True):
    """(i, j) arrays of the linked pairs; asserts that no candidate pair lies within 1e-9 b^2 of the threshold"""
    from scipy.spatial import cKDTree
    p = wrapped(pos, box) if box is not None else np.asarray(pos)
    if box is not None:
        t = cKDTree(np.mod(p.astype("f8"), np.asarray(box, "f8")), boxsize=np.asarray(box, "f8"))
    else:
        t = cKDTree(p.astype("f8"))
    cand = t.query_pairs(b * (1 + 1e-6) + 1e-12, output_type="ndarray")
    if len(cand) == 0:
        return np.zeros(0, "i8"), np.zeros(0, "i8")
    d2 = _d2(p[cand[:, 0]], p[cand[:, 1]], box)
    if check_margin:
        assert not np.any(np.abs(d2 - b * b) < 1e-9 * b * b), "a pair separation is too close to the linking length"
    keep = d2 <= b * b
    return cand[keep, 0], cand[keep, 1]


def minid(pos, b, box=None, check_margin=True):
    """smallest row of every particle's group"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    n = len(pos)
    i, j = friend_pairs(pos, b, box, check_margin)
    g = coo_matrix((np.ones(len(i)), (i, j)), shape=(n, n))
    _, comp = connected_components(g, directed=False)
    first = np.full(comp.max() + 1 if n else 0, n, "i8")
    np.minimum.at(first, comp, np.arange(n))
    return first[comp]


def labels_from_minid(mid, nmin):
    ids, inv, cnt = np.unique(mid, return_inverse=True, return_counts=True)
    big = cnt > nmin
    order = np.lexsort((ids[big], -cnt[big]))
    lab = np.zeros(len(ids), "i8")
    lab[np.nonzero(big)[0][order]] = np.arange(1, big.sum() + 1)
    return lab[inv]


def fof_labels(pos, b, nmin, box=None, check_margin=True):
    return labels_from_minid(minid(pos, b, box, check_margin), nmin)


def centerofmass(label, pos, nlab, box=None):
    pos = np.asarray(pos, "f8")
    N = np.bincount(label, minlength=nlab).astype("f8")
    if box is None:
        s = np.zeros((nlab, 3))
        np.add.at(s, label, pos)
        return s / N[:, None]
    L = np.asarray(box, "f8")
    pmin = np.full((nlab, 3), np.inf)
    np.minimum.at(pmin, label, pos)
    d = pos - pmin[label]
    d = np.where(d < -0.5 * L, d + L, d)
    d = np.where(d >= 0.5 * L, d - L, d)
    s = np.zeros((nlab, 3))
    np.add.at(s, label, d)
    return np.mod(pmin + s / N[:, None], L)


def features(label, pos, vel, box=None, peak=None):
    """the find_features columns in float64 (row 0: the particles of label 0)"""
    nlab = int(label.max()) + 1
    out = dict(Length=np.bincount(label, minlength=nlab), CMPosition=centerofmass(label, pos, nlab, box),
               CMVelocity=centerofmass(label, vel, nlab, None))
    out["Length"][0] = 0
    if peak is not None:
        dmax = np.full(nlab, -np.inf)
        np.maximum.at(dmax, label, np.asarray(peak, "f8"))
        sel = np.asarray(peak, "f8") >= dmax[label]
        out["PeakPosition"] = centerofmass(label[sel], np.asarray(pos)[sel], nlab, box)
        out["PeakVelocity"] = centerofmass(label[sel], np.asarray(vel)[sel], nlab, None)
    return out


def clustered_catalogue(seed, box, n_bg, clump_sizes, clump_scale, dtype="f8", periodic=True):
    """(pos, vel, peak): a uniform background of n_bg particles plus gaussian clumps of the given sizes (the test
    catalogues of the FOF fixtures and of the reference pinning test)"""
    rng = np.random.RandomState(seed)
    box = np.asarray(box, "f8")
    parts = [rng.uniform(size=(n_bg, 3)) * box]
    for s in clump_sizes:
        c = rng.uniform(size=3) * box
        parts.append(c + rng.normal(scale=clump_scale, size=(s, 3)))
    pos = np.concatenate(parts)
    if periodic:
        pos = np.mod(pos, box)
    pos = pos.astype(dtype)
    vel = rng.normal(size=pos.shape).astype(dtype)
    peak = rng.uniform(size=len(pos))
    return pos, vel, peak


def fixture_cases():
    """name -> (pos, vel, peak, box or None, b, nmin) of the tests/golden/fof_*.npz fixtures"""
    out = {}
    # distinct clump sizes above nmin over a sparse background: no two groups of label > 0 share a size
    pos, vel, peak = clustered_catalogue(1, [64.] * 3, 1500, list(range(25, 85, 3)), 0.05)
    out["distinct"] = (pos, vel, peak, [64.] * 3, 0.3, 20)
    pos, vel, peak = clustered_catalogue(2, [64.] * 3, 8000, [int(v) for v in np.random.RandomState(3).randint(5, 80, 60)],
                                         0.4, dtype="f4")
    out["clustered_f4"] = (pos, vel, peak, [64.] * 3, 0.45, 5)
    pos, vel, peak = clustered_catalogue(4, [40., 24., 16.], 2000, list(range(12, 72, 3)), 0.08)
    out["noncubic"] = (pos, vel, peak, [40., 24., 16.], 0.35, 10)
    pos, vel, peak = clustered_catalogue(5, [50.] * 3, 1500, list(range(15, 90, 3)), 0.08, periodic=False)
    out["nonperiodic"] = (pos - 25., vel, peak, None, 0.35, 10)
    return out
