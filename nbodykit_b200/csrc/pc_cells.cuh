// The neighbour-cell walk shared by the pair counts (paircount.cu) and the three-point function (threeptcf.cu): the
// cell-grid geometry, the per-axis stencil (wrapped when periodic, or every cell once when the periodic stencil wraps
// onto itself), the conservative gap of cells `delta` apart, and the search of a cell key in a key-sorted cell table.
#pragma once

#include "common.cuh"

struct PcGeom {
    double box[3];      // period (periodic) / extent of the cell grid (non-periodic)
    double cs[3];       // cell side
    double tol[3];      // how far a row may sit outside its cell after rounding (>= 2x the worst case)
    long long nc[3];    // cells per axis
    long long reach[3]; // largest cell-index difference of a pair within s_max
    int periodic;
    int mode;           // NBK_PC_1D / 2D / PROJECTED / SURVEY_2D / SURVEY_PROJECTED / ANGULAR
    int nb;             // bins along the first dimension (edges: nb + 1)
    int n2;             // bins along the second dimension (mu or pi; 1 in '1d' and 'angular')
    double thr_xy;      // skip a column when its smallest squared transverse gap reaches this
    double thr_sph;     // all but box 'projected': skip a cell when its smallest squared gap reaches this
    double pimax;       // 'projected': pairs need |dc| < pimax
};

// the smallest distance along an axis between rows of cells `delta` apart (a lower bound with margin)
static __device__ __forceinline__ double axis_gap(long long delta, int d, const PcGeom &g) {
    double v = (double)(delta - 1) * g.cs[d] - g.tol[d];
    return delta <= 1 || v < 0.0 ? 0.0 : v;
}

// cells of an axis within `r` of cell i: as offsets lo..hi (wrapped when periodic), or every cell once when the periodic
// stencil wraps onto itself (then delta is the minimum image)
struct PcAxis { long long lo, hi; bool all; };
static __device__ __forceinline__ PcAxis pc_axis(long long i, long long r, int d, const PcGeom &g) {
    PcAxis a;
    a.all = g.periodic && 2 * r + 1 >= g.nc[d];
    if (a.all) { a.lo = 0; a.hi = g.nc[d] - 1; }
    else if (g.periodic) { a.lo = i - r; a.hi = i + r; }
    else { a.lo = i - r < 0 ? 0 : i - r; a.hi = i + r > g.nc[d] - 1 ? g.nc[d] - 1 : i + r; }
    return a;
}
static __device__ __forceinline__ long long pc_wrap(long long v, long long n) { return v < 0 ? v + n : (v >= n ? v - n : v); }
// cell-index distance of offset cell cc (unwrapped) from i; the minimum image when the axis is visited whole
static __device__ __forceinline__ long long pc_delta(long long cc, long long i, bool all, long long n) {
    long long d = cc > i ? cc - i : i - cc;
    if (all && n - d < d) d = n - d;
    return d;
}

static __device__ __forceinline__ int64_t pc_lower_bound(const long long *ck, int64_t n, long long key) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        int64_t mid = (lo + hi) >> 1;
        if (ck[mid] < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}
