"""
TEST INFRASTRUCTURE -- CPU restatement of the fiber-collision contract (nbodykit_b200/algorithms/fibercollisions.py,
DESIGN.md 4.11); pinned against the reference's own code by tests/test_oracle_fibercollisions_reference.py
(oracle/fibercollisions_refload.py).

Groups: FOF labels of the positions (oracle/fof_oracle.py, periodic box 2.2, nmin 1).  A group of 2 loses the chosen one
of its two members, whose neighbour is the other.  In a group of 3 or more, members collide when
d = sqrt((dx^2 + dy^2) + dz^2) <= rad in double from the positions cast to float32; the greedy removes, among the alive
members with the most alive colliders (n_coll) and then the fewest n_coll summed over their alive colliders (n_other),
the chosen candidate, until one member is left; a removed member is collided when its n_coll > 0.  A collided member's
neighbour is the nearest uncollided member of its group by d, the first in member order on a tie.

The chooser `choose(g, step, k)` returns which of the k candidates (in member order) removal `step` of the group whose
smallest row is g takes.  `hash_chooser(seed)` is the package's rule; `numpy_chooser()` draws `numpy.random.choice` from
NumPy's global generator, as the reference does.  Member order: ascending row ('row') or the reference's structured sort,
byte-wise (memcmp) in the three float32 positions as stored, then the row ('reference'): NumPy orders the
float32 subarray field of the reference's structured `sort(order=['Label'])` by its bytes, not by value.
"""
import numpy as np

BOX = 2.2
_M = (1 << 64) - 1


def _splitmix(z):
    z = (z + 0x9E3779B97F4A7C15) & _M
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M
    return z ^ (z >> 31)


def hash_chooser(seed):
    def choose(g, step, k):
        h = _splitmix(_splitmix(_splitmix(int(seed)) ^ int(g)) ^ int(step))
        return ((h >> 32) * int(k)) >> 32
    return choose


def numpy_chooser():
    def choose(g, step, k):
        return int(np.random.choice(np.arange(k)))
    return choose


def unit_sphere(ra, dec, degrees=True):
    """SkyToUnitSphere + 1.1 in float64"""
    ra, dec = np.asarray(ra, "f8"), np.asarray(dec, "f8")
    if degrees:
        ra, dec = np.deg2rad(ra), np.deg2rad(dec)
    return np.stack([np.cos(dec) * np.cos(ra), np.cos(dec) * np.sin(ra), np.sin(dec)], axis=-1) + 1.1


def fof_labels(pos, rad, check_margin=True):
    from . import fof_oracle
    return fof_oracle.fof_labels(pos, rad, 1, box=[BOX] * 3, check_margin=check_margin)


def _dist(a, b):
    """d from float32 positions, in double"""
    d = np.asarray(a, "f8") - np.asarray(b, "f8")
    return np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])


def collision_lists(p4, rad):
    """per member (local index), its colliders"""
    n = len(p4)
    if n <= 256:
        d = _dist(p4[:, None, :], p4[None, :, :])
        np.fill_diagonal(d, np.inf)
        return [np.nonzero(d[i] <= rad)[0] for i in range(n)]
    from scipy.spatial import cKDTree
    cand = cKDTree(p4.astype("f8")).query_pairs(rad * (1 + 1e-6) + 1e-12, output_type="ndarray")
    keep = _dist(p4[cand[:, 0]], p4[cand[:, 1]]) <= rad
    i, j = cand[keep, 0], cand[keep, 1]
    a, b = np.concatenate([i, j]), np.concatenate([j, i])
    order = np.lexsort((b, a))
    a, b = a[order], b[order]
    starts = np.searchsorted(a, np.arange(n + 1))
    return [b[starts[k]:starts[k + 1]] for k in range(n)]


def greedy(p4, rad, choose, g, full=True):
    """(collided bool per member, forced: no removal of a collider had more than one candidate, collider removals).
    full=True runs until one member is left (every removal draws from the chooser); else it stops at the first removal
    without a collider, which gives the same result"""
    N = len(p4)
    adj = collision_lists(p4, rad)
    ncoll = np.array([len(a) for a in adj], "i8")
    nother = np.array([ncoll[a].sum() for a in adj], "i8")
    alive = np.ones(N, bool)
    coll = np.zeros(N, bool)
    forced = True
    step = 0
    while alive.sum() > 1:
        idx = np.nonzero(alive)[0]
        M = ncoll[idx].max()
        if M == 0 and not full:
            break
        cands = idx[ncoll[idx] == M]
        cands = cands[nother[cands] == nother[cands].min()]
        c = cands[choose(g, step, len(cands))]
        if M > 0:
            coll[c] = True
            forced = forced and len(cands) == 1
        alive[c] = False
        aj = adj[c][alive[adj[c]]]
        ncoll[aj] -= 1
        nother[aj] -= M
        if len(aj):
            ak = np.concatenate([adj[j] for j in aj])
            np.subtract.at(nother, ak[alive[ak]], 1)
        step += 1
    return coll, forced


def assign(pos, label, rad, choose, order="row", full=True):
    """(Collided i4, NeighborID i8, forced bool) per row of `pos` (any float dtype; cast to float32 for the distances)"""
    pos = np.asarray(pos)
    label = np.asarray(label)
    n = len(label)
    p4 = pos.astype("f4")
    collided = np.zeros(n, "i4")
    neighbor = np.full(n, -1, "i8")
    forced = np.zeros(n, bool)
    rows = np.nonzero(label > 0)[0]
    rows = rows[np.argsort(label[rows], kind="stable")]
    bounds = np.nonzero(np.diff(label[rows]))[0] + 1
    for mem in np.split(rows, bounds) if len(rows) else []:
        if order == "reference":
            b = np.ascontiguousarray(p4[mem]).view("u1").reshape(len(mem), 12)
            mem = mem[np.lexsort((mem,) + tuple(b[:, k] for k in range(11, -1, -1)))]
        g = int(mem.min())
        if len(mem) == 2:
            c = choose(g, 0, 2)
            collided[mem[c]] = 1
            neighbor[mem[c]] = mem[1 - c]
            continue
        q = p4[mem]
        coll, f = greedy(q, rad, choose, g, full)
        forced[mem] = f
        unc = np.nonzero(~coll)[0]
        for i in np.nonzero(coll)[0]:
            collided[mem[i]] = 1
            neighbor[mem[i]] = mem[unc[np.argmin(_dist(q[i][None, :], q[unc]))]]
    return collided, neighbor, forced


def fiber_collisions(pos, rad, seed, check_margin=True):
    """(Label, Collided, NeighborID) of the package's contract for the positions `pos` (unit sphere + 1.1)"""
    label = fof_labels(pos, rad, check_margin)
    c, nb, _ = assign(pos, label, rad, hash_chooser(seed), order="row", full=False)
    return label, c, nb


def check_invariants(pos, label, collided, neighbor, rad):
    """no two uncollided members of a multiplet collide; every collided member of a multiplet collides with a member
    that was alive when it was removed (checked as: it has a collider); NeighborID is the nearest uncollided member"""
    p4 = np.asarray(pos).astype("f4")
    rows = np.nonzero(label > 0)[0]
    for lab in np.unique(label[rows]):
        mem = np.nonzero(label == lab)[0]
        d = _dist(p4[mem][:, None, :], p4[mem][None, :, :])
        np.fill_diagonal(d, np.inf)
        c = collided[mem].astype(bool)
        assert (~c).any()
        if len(mem) > 2:
            assert not (d[np.ix_(~c, ~c)] <= rad).any()
            assert ((d[c] <= rad).sum(axis=1) >= 1).all()
        else:
            assert c.sum() == 1
        unc = mem[~c]
        for k in np.nonzero(c)[0]:
            dd = d[k][~c]
            assert neighbor[mem[k]] == unc[np.argmin(dd)]
        assert (neighbor[mem[~c]] == -1).all()
