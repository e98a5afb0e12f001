"""
TEST INFRASTRUCTURE -- a NumPy / scipy restatement of the KDDensity contract (DESIGN.md 4.10).

q = pos / L in the positions' own dtype (an in-place divide by a float64 BoxSize array, so float32 positions give
f4(f8(x) / L)), then `q %= 1` in that dtype; a q of 1.0 becomes 0.0.  d is the 8th smallest distance from each row to
all rows, itself included, from scipy's periodic cKDTree on q as float64 (its per-axis wrap and sum of squares are the
contract's), inf with fewer than 8 rows; density = 1 / (d^3 V).
"""
import numpy
from scipy.spatial import cKDTree

K = 8


def unit(pos, L):
    """the unit coordinates of `pos` in a cubic box of side L, in the positions' dtype"""
    q = numpy.array(pos, copy=True)
    q[...] /= numpy.array([L, L, L], dtype='f8')
    q %= 1
    q[q == 1] = 0
    return q


def distance(pos, L):
    """d of every row"""
    q = unit(pos, L).astype('f8')
    if len(q) == 0:
        return numpy.zeros(0)
    d, _ = cKDTree(q, boxsize=1.0).query(q, k=[K])
    return d[:, 0]


def density(pos, L):
    """(d, density) of every row"""
    d = distance(pos, L)
    with numpy.errstate(divide='ignore'):
        return d, 1 / (d ** 3 * numpy.array([L, L, L], dtype='f8').prod())
