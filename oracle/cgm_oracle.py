"""
TEST INFRASTRUCTURE -- a float64 NumPy restatement of the CylindricalGroups contract (DESIGN.md 4.9).

Priority from `numpy.lexsort` (ties by ascending row, -0.0 == 0.0), candidate pairs from scipy's cKDTree at
rmax (1 + 1e-9), the exact link test of the contract on each candidate, then the sequential greedy: the
highest-priority unassigned row becomes a central and every unassigned row linked to it its satellite.
"""
import numpy
from scipy.spatial import cKDTree


def priority(keys, n, reverse=False):
    """position of every row in the lexicographic order of `keys` (first key primary), ties by ascending row"""
    if not keys:
        return numpy.arange(n, dtype='i8')
    cols = []
    for k in keys:
        k = numpy.asarray(k)
        if k.dtype.kind == 'f':
            k = numpy.where(k == 0, 0.0, k.astype('f8'))
        # dense ranks: descending order is the ascending order of negated ranks, for any dtype
        _, r = numpy.unique(k, return_inverse=True)
        r = r.reshape(-1).astype('i8')
        cols.append(-r if reverse else r)
    order = numpy.lexsort([numpy.arange(n)] + cols[::-1])
    prio = numpy.empty(n, dtype='i8')
    prio[order] = numpy.arange(n)
    return prio


def wrap(pos, box):
    """numpy's `pos % L` in the positions' own dtype"""
    return pos % numpy.asarray(box, dtype=pos.dtype)


def linked(xa, xb, rperp, rpar, los=None, box=None):
    """the link of rows a (the higher priority) and b, vectorised over (m, 3) float64 arrays"""
    d = [xa[:, k] - xb[:, k] for k in range(3)]
    if box is not None:
        for k in range(3):
            L = float(box[k])
            d[k] = numpy.where(d[k] > L * 0.5, d[k] - L, numpy.where(d[k] <= -L * 0.5, d[k] + L, d[k]))
    dx, dy, dz = d
    dr2 = (dx * dx + dy * dy) + dz * dz
    with numpy.errstate(invalid='ignore', divide='ignore'):
        if los is not None:
            lx, ly, lz = [float(v) for v in los]
            t = (dx * lx + dy * ly) + dz * lz
            rlos2 = t * t
            ok = numpy.ones(len(dx), dtype=bool)
        else:
            cx, cy, cz = [0.5 * (xa[:, k] + xb[:, k]) for k in range(3)]
            den = (cx * cx + cy * cy) + cz * cz
            t = (dx * cx + dy * cy) + dz * cz
            ok = den > 0
            rlos2 = numpy.where(ok, (t * t) / numpy.where(ok, den, 1.0), numpy.inf)
        rsky2 = numpy.abs(dr2 - rlos2)
    rperp2, rpar2 = float(rperp) * float(rperp), float(rpar) * float(rpar)
    return ok & (rsky2 <= rperp2) & (rlos2 <= rpar2)


def candidates(pos, rmax, box=None):
    """(i, j) index arrays of every pair within rmax (1 + 1e-9), i < j"""
    p = numpy.asarray(pos, dtype='f8')
    if box is not None:
        L = numpy.asarray(box, dtype='f8')
        p = numpy.where(p >= L, p - L, p)
        tree = cKDTree(p, boxsize=L)
    else:
        tree = cKDTree(p)
    pairs = tree.query_pairs(rmax * (1 + 1e-9), output_type='ndarray')
    if len(pairs) == 0:
        return numpy.zeros(0, 'i8'), numpy.zeros(0, 'i8')
    return pairs[:, 0].astype('i8'), pairs[:, 1].astype('i8')


def cgm(pos, keys, rperp, rpar, los=None, periodic=False, BoxSize=None):
    """(cgm_type u4, cgm_haloid i8, num_cgm_sats i8, priority) of every row"""
    pos = numpy.asarray(pos)
    n = len(pos)
    box = numpy.ones(3) * numpy.asarray(BoxSize, dtype='f8') if periodic else None
    if periodic:
        pos = wrap(pos, box)
    x = pos.astype('f8')
    prio = priority(keys, n)
    rmax = (float(rperp) ** 2 + float(rpar) ** 2) ** 0.5
    i, j = candidates(x, rmax, box)
    hi = numpy.where(prio[i] > prio[j], i, j)
    lo = numpy.where(prio[i] > prio[j], j, i)
    ok = linked(x[hi], x[lo], rperp, rpar, los, box)
    hi, lo = hi[ok], lo[ok]
    # per row, its linked rows of higher priority
    o = numpy.argsort(lo, kind='stable')
    hi, lo = hi[o], lo[o]
    start = numpy.searchsorted(lo, numpy.arange(n + 1))
    state = numpy.zeros(n, dtype='i1')              # 1 central, 2 satellite
    cen_of = numpy.full(n, -1, dtype='i8')
    for r in numpy.argsort(-prio, kind='stable'):
        up = hi[start[r]:start[r + 1]]
        cens = up[state[up] == 1]
        if len(cens):
            state[r] = 2
            cen_of[r] = cens[numpy.argmax(prio[cens])]
        else:
            state[r] = 1
            cen_of[r] = r
    is_cen = state == 1
    cen_prio = numpy.sort(prio[is_cen])[::-1]
    haloid_by_prio = numpy.full(n, -1, dtype='i8')
    haloid_by_prio[cen_prio] = numpy.arange(len(cen_prio))
    haloid = haloid_by_prio[prio[cen_of]] if n else numpy.zeros(0, 'i8')
    nsat = numpy.zeros(n, dtype='i8')
    sat = ~is_cen
    numpy.add.at(nsat, cen_of[sat], 1)
    return (state == 2).astype('u4'), haloid.astype('i8'), nsat, prio
