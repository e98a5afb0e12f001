// Friends-of-friends groups (nbodykit/algorithms/fof.py: the kdcount tree FOF of `_fof_local`, the `_fof_merge` fixed
// point and the per-label reductions of `centerofmass` / `fof_catalog`) on cell keys instead of a kd-tree.
//   nbk_fof_cell_keys   : 64-bit key of the cell (side <= b / sqrt 3) of every particle
//   nbk_fof_sorted_pos  : positions gathered into key order, wrapped with numpy's `pos % L` semantics when periodic
//   nbk_fof_sort        : stable radix sort of 64-bit cell keys / 32-bit labels with 32-bit row indices (cub, double
//                         buffered: 12 or 8 bytes per row of scratch, nothing else)
//   nbk_fof_compact_*   : count, then write the table of the occupied cells (first row, key) of the key-sorted rows
//   nbk_fof_link        : union-find over occupied cells: every cell is internally linked; a pair of cells within reach
//                         is united at the first particle pair with d^2 <= b^2; roots are the cells holding the smallest
//                         global id of their component
//   nbk_fof_finalize    : per row: root cell and minid (smallest global id of the group)
//   nbk_fof_lower       : lower every local component to the smallest minid any of its rows carries (multi-rank merge)
//   nbk_fof_root_counts : rows per root cell
//   nbk_fof_label_rows  : per row label from the per-cell label table
//   nbk_fof_segment_reduce : fixed-order segmented min / max / (wrapped) sums over rows ordered by label
// Distances: d^2 = (dx^2 + dy^2) + dz^2 in double from the stored (wrapped) positions, per-axis |d| -> min(|d|, L - |d|)
// when periodic.  The file is compiled with --fmad=false: no contraction may change a link decision.
#include "common.cuh"

#include <math.h>

#include <cub/device/device_radix_sort.cuh>

#define FOF_MAX_CELLS_PER_AXIS (1ll << 21)

struct FofGeom {
    double box[3];     // period (periodic) / extent of the cell grid (non-periodic)
    double org[3];     // grid origin (non-periodic)
    double inv[3];     // ncell / box
    long long nc[3];   // cells per axis
    long long reach[3];  // largest cell-index difference of a linked pair, per axis
    int full[3];       // periodic axis the reach wraps onto itself: visit each of its cells once
    int periodic;
    double b2;
};

static __device__ __forceinline__ float np_fmod(float x, float L) { return fmodf(x, L); }
static __device__ __forceinline__ double np_fmod(double x, double L) { return fmod(x, L); }

// numpy's float `x % L` (npy_divmod): fmod, then + L when the remainder is negative (may round up to L itself)
template <typename T>
static __device__ __forceinline__ T np_mod(T x, T L) {
    T r = np_fmod(x, L);
    if (r != (T)0 && r < (T)0) r += L;
    return r;
}

// Every row must lie inside its cell on every axis (up to rounding), because FOF links every pair of one cell unseen.
// A periodic row at q >= nc sits at or above the period L: an f4 row wrapped onto L_f4 > L, or an f8 row that `x % L`
// rounded up to L.  Its minimum image is L_f4 - L (or 0) above 0, so it belongs to cell 0; clamping it into cell
// nc - 1 would put it up to cs + (L_f4 - L) from that cell's lower corner.
template <typename T>
static __device__ __forceinline__ long long cell_of(T p, int d, const FofGeom &g) {
    double q = g.periodic ? (double)p * g.inv[d] : ((double)p - g.org[d]) * g.inv[d];
    long long c = (long long)floor(q);
    if (c >= g.nc[d]) return g.periodic ? 0 : g.nc[d] - 1;
    return c < 0 ? 0 : c;
}

template <typename T>
__global__ void __launch_bounds__(256) k_fof_keys(const T *__restrict__ pos, int64_t n, FofGeom g, long long *__restrict__ keys) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        long long c[3];
#pragma unroll
        for (int d = 0; d < 3; d++) {
            T p = pos[3 * i + d];
            if (g.periodic) p = np_mod(p, (T)g.box[d]);
            c[d] = cell_of(p, d, g);
        }
        keys[i] = (c[0] * g.nc[1] + c[1]) * g.nc[2] + c[2];
    }
}

template <typename T>
__global__ void __launch_bounds__(256) k_fof_sorted_pos(const T *__restrict__ pos, int64_t n, const unsigned *__restrict__ perm,
                                                        FofGeom g, T *__restrict__ spos) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        int64_t r = perm[i];
#pragma unroll
        for (int d = 0; d < 3; d++) {
            T p = pos[3 * r + d];
            spos[3 * i + d] = g.periodic ? np_mod(p, (T)g.box[d]) : p;
        }
    }
}

// ---- compaction of the occupied cells: tiles of FOF_TILE sorted keys, counted, scanned, written in order
#define FOF_TILE 4096
#define FOF_CB 256

static __device__ __forceinline__ bool is_first(const long long *k, int64_t i) { return i == 0 || k[i] != k[i - 1]; }

__global__ void __launch_bounds__(FOF_CB) k_fof_tile_count(const long long *__restrict__ keys, int64_t n, long long *__restrict__ tiles) {
    int64_t t0 = (int64_t)blockIdx.x * FOF_TILE;
    int cnt = 0;
    for (int s = 0; s < FOF_TILE; s += FOF_CB) {
        int64_t i = t0 + s + threadIdx.x;
        cnt += __syncthreads_count(i < n && is_first(keys, i));
    }
    if (threadIdx.x == 0) tiles[blockIdx.x] = cnt;
}

// exclusive scan of the tile counts in one block; tiles[ntiles] = number of cells
__global__ void __launch_bounds__(1024) k_fof_tile_scan(long long *__restrict__ tiles, int64_t ntiles, long long *__restrict__ ncells) {
    __shared__ long long part[1024];
    int64_t per = (ntiles + blockDim.x - 1) / blockDim.x;
    int64_t a = threadIdx.x * per, b = min(a + per, ntiles);
    long long s = 0;
    for (int64_t i = a; i < b; i++) s += tiles[i];
    part[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        long long acc = 0;
        for (int i = 0; i < (int)blockDim.x; i++) { long long v = part[i]; part[i] = acc; acc += v; }
        tiles[ntiles] = acc;
        *ncells = acc;
    }
    __syncthreads();
    long long acc = part[threadIdx.x];
    for (int64_t i = a; i < b; i++) { long long v = tiles[i]; tiles[i] = acc; acc += v; }
}

__global__ void __launch_bounds__(FOF_CB) k_fof_tile_write(const long long *__restrict__ keys, int64_t n, const long long *__restrict__ tiles,
                                                           int64_t ntiles, unsigned *__restrict__ cell_start, long long *__restrict__ cell_key) {
    __shared__ int wsum[FOF_CB / 32];
    __shared__ long long base;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (threadIdx.x == 0) base = tiles[blockIdx.x];
    if (blockIdx.x == 0 && threadIdx.x == 0) cell_start[tiles[ntiles]] = (unsigned)n;
    __syncthreads();
    int64_t t0 = (int64_t)blockIdx.x * FOF_TILE;
    for (int s = 0; s < FOF_TILE; s += FOF_CB) {
        int64_t i = t0 + s + threadIdx.x;
        bool f = i < n && is_first(keys, i);
        unsigned m = __ballot_sync(0xffffffffu, f);
        if (lane == 0) wsum[w] = __popc(m);
        __syncthreads();
        int before = 0, total = 0;
        for (int k = 0; k < FOF_CB / 32; k++) { if (k < w) before += wsum[k]; total += wsum[k]; }
        if (f) {
            long long dst = base + before + __popc(m & ((1u << lane) - 1u));
            cell_start[dst] = (unsigned)i;
            cell_key[dst] = keys[i];
        }
        __syncthreads();
        if (threadIdx.x == 0) base += total;
        __syncthreads();
    }
}

// ---- union-find over cells (lock-free hooking: the root with the larger smallest-id hooks under the other)
static __device__ __forceinline__ unsigned uf_find(unsigned *parent, unsigned x) {
    volatile unsigned *vp = parent;
    while (true) {
        unsigned p = vp[x];
        if (p == x) return x;
        unsigned gp = vp[p];
        if (gp == p) return p;
        vp[x] = gp;       // path halving: gp is an ancestor of x whatever else runs
        x = gp;
    }
}

static __device__ __forceinline__ void uf_unite(unsigned *parent, const long long *cmin, unsigned a, unsigned b) {
    while (true) {
        a = uf_find(parent, a);
        b = uf_find(parent, b);
        if (a == b) return;
        if (cmin[a] < cmin[b]) { unsigned t = a; a = b; b = t; }
        if (atomicCAS(&parent[a], a, b) == a) return;
    }
}

__global__ void __launch_bounds__(256) k_fof_init(const unsigned *__restrict__ cell_start, int64_t ncells, const unsigned *__restrict__ perm,
                                                  const long long *__restrict__ gid, long long gid_base, unsigned *__restrict__ parent,
                                                  long long *__restrict__ cmin) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < ncells; c += stride) {
        long long m = LLONG_MAX;
        for (long long j = cell_start[c]; j < cell_start[c + 1]; j++) {
            long long r = (long long)perm[j];
            long long id = gid ? gid[r] : gid_base + r;
            m = id < m ? id : m;
        }
        parent[c] = (unsigned)c;
        cmin[c] = m;
    }
}

template <typename T>
static __device__ __forceinline__ double fof_d2(const T *a, const T *b, const FofGeom &g) {
    double s[3];
#pragma unroll
    for (int d = 0; d < 3; d++) {
        double x = fabs((double)a[d] - (double)b[d]);
        if (g.periodic) x = fmin(x, g.box[d] - x);
        s[d] = x * x;
    }
    return (s[0] + s[1]) + s[2];
}

// lower_bound of `key` in the sorted cell keys
static __device__ __forceinline__ int64_t cell_lower_bound(const long long *ck, int64_t ncells, long long key) {
    int64_t lo = 0, hi = ncells;
    while (lo < hi) {
        int64_t mid = (lo + hi) >> 1;
        if (ck[mid] < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// the distinct cell coordinates within reach of coordinate i on axis d (count, first, wrap)
struct AxisSet { long long lo, hi; };
static __device__ __forceinline__ AxisSet axis_set(long long i, int d, const FofGeom &g) {
    AxisSet s;
    if (g.full[d]) { s.lo = 0; s.hi = g.nc[d] - 1; }
    else if (g.periodic) { s.lo = i - g.reach[d]; s.hi = i + g.reach[d]; }
    else { s.lo = max(0ll, i - g.reach[d]); s.hi = min(g.nc[d] - 1, i + g.reach[d]); }
    return s;
}
static __device__ __forceinline__ long long wrapc(long long v, long long n) { return v < 0 ? v + n : (v >= n ? v - n : v); }

template <typename T>
__global__ void __launch_bounds__(128) k_fof_link(const T *__restrict__ spos, const unsigned *__restrict__ cell_start,
                                                  const long long *__restrict__ ckey, int64_t ncells, FofGeom g,
                                                  unsigned *__restrict__ parent, const long long *__restrict__ cmin) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const long long nyz = g.nc[1] * g.nc[2];
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < ncells; c += stride) {
        const long long key = ckey[c];
        const long long ix = key / nyz, iy = (key / g.nc[2]) % g.nc[1], iz = key % g.nc[2];
        const long long c0 = cell_start[c], c1 = cell_start[c + 1];
        AxisSet sx = axis_set(ix, 0, g), sy = axis_set(iy, 1, g), sz = axis_set(iz, 2, g);
        for (long long xx = sx.lo; xx <= sx.hi; xx++) {
            const long long x = g.periodic ? wrapc(xx, g.nc[0]) : xx;
            for (long long yy = sy.lo; yy <= sy.hi; yy++) {
                const long long y = g.periodic ? wrapc(yy, g.nc[1]) : yy;
                const long long row = (x * g.nc[1] + y) * g.nc[2];
                // the z range as up to two contiguous key ranges
                long long r0[2], r1[2];
                int nr = 0;
                if (sz.lo < 0) { r0[nr] = sz.lo + g.nc[2]; r1[nr++] = g.nc[2] - 1; r0[nr] = 0; r1[nr++] = sz.hi; }
                else if (sz.hi >= g.nc[2]) { r0[nr] = sz.lo; r1[nr++] = g.nc[2] - 1; r0[nr] = 0; r1[nr++] = sz.hi - g.nc[2]; }
                else { r0[nr] = sz.lo; r1[nr++] = sz.hi; }
                for (int q = 0; q < nr; q++) {
                    long long k0 = row + r0[q], k1 = row + r1[q];
                    if (k1 <= key) continue;          // each unordered pair of cells once: the partner has the larger key
                    if (k0 <= key) k0 = key + 1;
                    for (int64_t d = cell_lower_bound(ckey, ncells, k0); d < ncells && ckey[d] <= k1; d++) {
                        if (uf_find(parent, (unsigned)c) == uf_find(parent, (unsigned)d)) continue;
                        const long long d0 = cell_start[d], d1 = cell_start[d + 1];
                        bool hit = false;
                        for (long long a = c0; a < c1 && !hit; a++) {
                            const T pa[3] = {spos[3 * a], spos[3 * a + 1], spos[3 * a + 2]};
                            for (long long bb = d0; bb < d1; bb++) {
                                if (fof_d2(pa, spos + 3 * bb, g) <= g.b2) { hit = true; break; }
                            }
                        }
                        if (hit) uf_unite(parent, cmin, (unsigned)c, (unsigned)d);
                    }
                }
            }
        }
    }
}

// after the link pass: parent[c] = root, read-only walks so that only roots are ever stored
__global__ void __launch_bounds__(256) k_fof_compress(unsigned *__restrict__ parent, int64_t ncells) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    volatile unsigned *vp = parent;
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < ncells; c += stride) {
        unsigned x = (unsigned)c, p = vp[x];
        while (p != x) { x = p; p = vp[x]; }
        vp[c] = x;
    }
}

__global__ void __launch_bounds__(256) k_fof_finalize(const unsigned *__restrict__ perm, const unsigned *__restrict__ cell_start,
                                                      int64_t ncells, const unsigned *__restrict__ parent,
                                                      const long long *__restrict__ cmin, unsigned *__restrict__ row_root,
                                                      long long *__restrict__ minid) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < ncells; c += stride) {
        unsigned r = parent[c];
        long long m = cmin[r];
        for (long long j = cell_start[c]; j < cell_start[c + 1]; j++) {
            const unsigned row = perm[j];
            row_root[row] = r;
            if (minid) minid[row] = m;
        }
    }
}

__global__ void __launch_bounds__(256) k_fof_fill_i64(long long *__restrict__ x, int64_t n, long long v) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) x[i] = v;
}

__global__ void __launch_bounds__(256) k_fof_root_min(const unsigned *__restrict__ row_root, int64_t n, const long long *__restrict__ v,
                                                      long long *__restrict__ rootmin) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        atomicMin(&rootmin[row_root[i]], v[i]);
}

__global__ void __launch_bounds__(256) k_fof_root_read(const unsigned *__restrict__ row_root, int64_t n, const long long *__restrict__ rootmin,
                                                       long long *__restrict__ minid, unsigned long long *__restrict__ changed) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int64_t nround = ((n + stride - 1) / stride) * stride;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nround; i += stride) {
        bool ch = false;
        if (i < n) {
            long long m = rootmin[row_root[i]];
            ch = m != minid[i];
            minid[i] = m;
        }
        unsigned b = __ballot_sync(0xffffffffu, ch);
        if ((threadIdx.x & 31) == 0 && b) atomicAdd(changed, (unsigned long long)__popc(b));
    }
}

__global__ void __launch_bounds__(256) k_fof_root_counts(const unsigned *__restrict__ row_root, int64_t n, unsigned long long *__restrict__ counts) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) atomicAdd(&counts[row_root[i]], 1ull);
}

template <typename LT>
__global__ void __launch_bounds__(256) k_fof_label_rows(const unsigned *__restrict__ row_root, int64_t n, const long long *__restrict__ cell_label,
                                                        LT *__restrict__ labels) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) labels[i] = (LT)cell_label[row_root[i]];
}

// ---- fixed-order segmented reductions over rows ordered by label.  Chunk k covers sorted rows
// [chunk_first[k], chunk_first[k+1]) of label chunk_label[k]; label l owns chunks [label_chunk[l], label_chunk[l+1]).
// Each chunk is reduced by one block in a fixed tree order into partial[k][4]; each label then folds its chunks in
// order.  ops (NBK_FOF_RED_*): MIN of a 3-vector column, MAX of a scalar column, SUM of a 3-vector column minus ref[l]
// (wrapped into [-L/2, L/2) when periodic) with the included-row count in slot 3; a `mask` column restricts MIN / SUM
// to rows with mask >= thresh[l] (the peak particles).
#define FOF_RB 256

template <typename T>
static __device__ __forceinline__ double ldv(const void *p, int64_t i) { return (double)((const T *)p)[i]; }
static __device__ __forceinline__ double ldcol(const void *p, int dt, int64_t i) { return dt == NBK_F4 ? ldv<float>(p, i) : ldv<double>(p, i); }

struct RedArgs {
    const void *col; int col_dt; const void *mask; int mask_dt; const double *thresh; const double *ref;
    int op, periodic; double box[3];
};

static __device__ __forceinline__ void red_ident(int op, double v[4]) {
    double id = op == NBK_FOF_RED_MIN ? INFINITY : (op == NBK_FOF_RED_MAX ? -INFINITY : 0.0);
    v[0] = v[1] = v[2] = id;
    v[3] = 0.0;
}
static __device__ __forceinline__ void red_comb(int op, double a[4], const double b[4]) {
    if (op == NBK_FOF_RED_MIN) { for (int k = 0; k < 3; k++) a[k] = fmin(a[k], b[k]); }
    else if (op == NBK_FOF_RED_MAX) { a[0] = fmax(a[0], b[0]); }
    else { for (int k = 0; k < 3; k++) a[k] += b[k]; }
    a[3] += b[3];
}

__global__ void __launch_bounds__(FOF_RB) k_fof_reduce_chunks(RedArgs A, const unsigned *__restrict__ order, const long long *__restrict__ chunk_first,
                                                             const long long *__restrict__ chunk_label, double *__restrict__ partial) {
    __shared__ double sh[FOF_RB][4];
    const int64_t k = blockIdx.x;
    const long long l = chunk_label[k];
    const double th = A.thresh ? A.thresh[l] : 0.0;
    double acc[4];
    red_ident(A.op, acc);
    for (long long j = chunk_first[k] + threadIdx.x; j < chunk_first[k + 1]; j += FOF_RB) {
        const long long r = (long long)order[j];
        if (A.mask && !(ldcol(A.mask, A.mask_dt, r) >= th)) continue;
        double v[4];
        if (A.op == NBK_FOF_RED_MAX) { v[0] = ldcol(A.col, A.col_dt, r); v[1] = v[2] = 0.0; }
        else {
            for (int d = 0; d < 3; d++) {
                double x = ldcol(A.col, A.col_dt, 3 * r + d);
                if (A.op == NBK_FOF_RED_SUM && A.ref) {
                    x = x - A.ref[3 * l + d];
                    if (A.periodic) {
                        double h = A.box[d] * 0.5;
                        if (x < -h) x += A.box[d];
                        else if (x >= h) x -= A.box[d];
                    }
                }
                v[d] = x;
            }
        }
        v[3] = 1.0;
        red_comb(A.op, acc, v);
    }
    for (int d = 0; d < 4; d++) sh[threadIdx.x][d] = acc[d];
    __syncthreads();
    for (int s = FOF_RB / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) {
            double a[4], b[4];
            for (int d = 0; d < 4; d++) { a[d] = sh[threadIdx.x][d]; b[d] = sh[threadIdx.x + s][d]; }
            red_comb(A.op, a, b);
            for (int d = 0; d < 4; d++) sh[threadIdx.x][d] = a[d];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0)
        for (int d = 0; d < 4; d++) partial[4 * k + d] = sh[0][d];
}

__global__ void __launch_bounds__(256) k_fof_reduce_labels(int op, const double *__restrict__ partial, const long long *__restrict__ label_chunk,
                                                           int64_t nlabels, double *__restrict__ out) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t l = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; l < nlabels; l += stride) {
        double acc[4];
        red_ident(op, acc);
        for (long long k = label_chunk[l]; k < label_chunk[l + 1]; k++) red_comb(op, acc, partial + 4 * k);
        for (int d = 0; d < 4; d++) out[4 * l + d] = acc[d];
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// the cell grid alone (box, origin, cell counts); b = 0 leaves reach / full / b2 unset (nbk_fof_grid_keys)
static int fof_grid(FofGeom &g, int periodic, const double *box, const double *origin, const int64_t *ncell, double b) {
    double cells = 1.0;
    for (int d = 0; d < 3; d++) {
        NBK_CHECK_ARG(isfinite(box[d]) && box[d] > 0, "fof: box side %d must be positive and finite (got %g)", d, box[d]);
        NBK_CHECK_ARG(ncell[d] >= 1 && ncell[d] <= FOF_MAX_CELLS_PER_AXIS, "fof: cell count %lld on axis %d out of range",
                      (long long)ncell[d], d);
        NBK_CHECK_ARG(periodic || (origin != nullptr && isfinite(origin[d])), "fof: non-periodic grids need a finite origin");
        cells *= (double)ncell[d];
        g.box[d] = box[d];
        g.org[d] = periodic ? 0.0 : origin[d];
        g.nc[d] = ncell[d];
        g.inv[d] = (double)ncell[d] / box[d];
        g.reach[d] = 0;
        g.full[d] = 0;
        if (b > 0) {
            double cs = box[d] / (double)ncell[d];
            NBK_CHECK_ARG(3.0 * cs * cs <= b * b, "fof: cells on axis %d are wider than b / sqrt(3)", d);
            g.reach[d] = (long long)floor(b / cs * (1.0 + 1e-12)) + 1;
            g.full[d] = periodic && 2 * g.reach[d] + 1 >= g.nc[d];
        }
    }
    NBK_CHECK_ARG(cells < 9.2e18, "fof: %g cells do not fit a 63-bit key", cells);
    g.periodic = periodic ? 1 : 0;
    g.b2 = b * b;
    return NBK_OK;
}

static int fof_geom(FofGeom &g, int periodic, const double *box, const double *origin, const int64_t *ncell, double b) {
    NBK_CHECK_ARG(box != nullptr && ncell != nullptr, "fof: box and cell counts are required");
    NBK_CHECK_ARG(b > 0 && isfinite(b), "fof: linking length must be positive and finite (got %g)", b);
    return fof_grid(g, periodic, box, origin, ncell, b);
}

#define FOF_CHECK_N(n) NBK_CHECK_ARG((n) >= 0 && (n) < (1ll << 32), "fof: row count %lld out of range", (long long)(n))
#define FOF_CHECK_DT(dt) NBK_CHECK_ARG((dt) == NBK_F4 || (dt) == NBK_F8, "fof: bad position dtype %d", (dt))

extern "C" int nbk_fof_cell_keys(const void *pos, int pos_dtype, int64_t n, int periodic, const double *box_host,
                                 const double *origin_host, const int64_t *ncell_host, double b, int64_t *keys, void *stream) {
    FOF_CHECK_DT(pos_dtype);
    FOF_CHECK_N(n);
    FofGeom g;
    int rc = fof_geom(g, periodic, box_host, origin_host, ncell_host, b);
    if (rc) return rc;
    if (n == 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    int grid = nbk_grid_for(n, 256, 8);
    if (pos_dtype == NBK_F4) k_fof_keys<float><<<grid, 256, 0, s>>>((const float *)pos, n, g, (long long *)keys);
    else k_fof_keys<double><<<grid, 256, 0, s>>>((const double *)pos, n, g, (long long *)keys);
    NBK_LAUNCHED();
    return NBK_OK;
}

// the keys of nbk_fof_cell_keys on a grid of any cell size (the pair counts choose cells from their largest separation)
extern "C" int nbk_fof_grid_keys(const void *pos, int pos_dtype, int64_t n, int periodic, const double *box_host,
                                 const double *origin_host, const int64_t *ncell_host, int64_t *keys, void *stream) {
    FOF_CHECK_DT(pos_dtype);
    FOF_CHECK_N(n);
    NBK_CHECK_ARG(box_host != nullptr && ncell_host != nullptr, "fof: box and cell counts are required");
    FofGeom g;
    int rc = fof_grid(g, periodic, box_host, origin_host, ncell_host, 0.0);
    if (rc) return rc;
    if (n == 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    int grid = nbk_grid_for(n, 256, 8);
    if (pos_dtype == NBK_F4) k_fof_keys<float><<<grid, 256, 0, s>>>((const float *)pos, n, g, (long long *)keys);
    else k_fof_keys<double><<<grid, 256, 0, s>>>((const double *)pos, n, g, (long long *)keys);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_fof_sorted_pos(const void *pos, int pos_dtype, int64_t n, const uint32_t *perm, int periodic,
                                  const double *box_host, void *sorted_pos, void *stream) {
    FOF_CHECK_DT(pos_dtype);
    FOF_CHECK_N(n);
    NBK_CHECK_ARG(box_host != nullptr, "fof: box is required");
    FofGeom g = {};
    for (int d = 0; d < 3; d++) {
        NBK_CHECK_ARG(isfinite(box_host[d]) && box_host[d] > 0, "fof: box side %d must be positive and finite", d);
        g.box[d] = box_host[d];
    }
    g.periodic = periodic ? 1 : 0;
    if (n == 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    int grid = nbk_grid_for(n, 256, 8);
    if (pos_dtype == NBK_F4) k_fof_sorted_pos<float><<<grid, 256, 0, s>>>((const float *)pos, n, (const unsigned *)perm, g, (float *)sorted_pos);
    else k_fof_sorted_pos<double><<<grid, 256, 0, s>>>((const double *)pos, n, (const unsigned *)perm, g, (double *)sorted_pos);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int64_t nbk_fof_compact_workspace(int64_t n) { return n < 0 ? -1 : (n + FOF_TILE - 1) / FOF_TILE + 1; }

extern "C" int nbk_fof_compact_count(const int64_t *sorted_keys, int64_t n, int64_t *work, int64_t work_len, int64_t *ncells,
                                     void *stream) {
    FOF_CHECK_N(n);
    NBK_CHECK_ARG(n >= 1, "fof_compact: needs at least one row");
    const int64_t ntiles = (n + FOF_TILE - 1) / FOF_TILE;
    NBK_CHECK_ARG(work_len >= ntiles + 1, "fof_compact: workspace of %lld entries, %lld needed", (long long)work_len,
                  (long long)(ntiles + 1));
    cudaStream_t s = (cudaStream_t)stream;
    k_fof_tile_count<<<(unsigned)ntiles, FOF_CB, 0, s>>>((const long long *)sorted_keys, n, (long long *)work);
    NBK_LAUNCHED();
    k_fof_tile_scan<<<1, 1024, 0, s>>>((long long *)work, ntiles, (long long *)ncells);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_fof_compact_write(const int64_t *sorted_keys, int64_t n, const int64_t *work, int64_t work_len,
                                     uint32_t *cell_start, int64_t *cell_key, void *stream) {
    FOF_CHECK_N(n);
    NBK_CHECK_ARG(n >= 1, "fof_compact: needs at least one row");
    const int64_t ntiles = (n + FOF_TILE - 1) / FOF_TILE;
    NBK_CHECK_ARG(work_len >= ntiles + 1, "fof_compact: workspace of %lld entries, %lld needed", (long long)work_len,
                  (long long)(ntiles + 1));
    k_fof_tile_write<<<(unsigned)ntiles, FOF_CB, 0, (cudaStream_t)stream>>>((const long long *)sorted_keys, n,
                                                                            (const long long *)work, ntiles,
                                                                            (unsigned *)cell_start, (long long *)cell_key);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int64_t nbk_fof_sort_workspace(int64_t n, int key_bytes) {
    if (n < 0 || n >= (1ll << 32) || (key_bytes != 4 && key_bytes != 8)) return -1;
    size_t bytes = 0;
    cub::DoubleBuffer<unsigned long long> k8(nullptr, nullptr);
    cub::DoubleBuffer<unsigned> k4(nullptr, nullptr), v(nullptr, nullptr);
    cudaError_t e = key_bytes == 8 ? cub::DeviceRadixSort::SortPairs(nullptr, bytes, k8, v, (int)n)
                                   : cub::DeviceRadixSort::SortPairs(nullptr, bytes, k4, v, (int)n);
    return e == cudaSuccess ? (int64_t)bytes : -1;
}

__global__ void __launch_bounds__(256) k_fof_iota(unsigned *__restrict__ v, int64_t n) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) v[i] = (unsigned)i;
}

extern "C" int nbk_fof_sort(void *keys, void *keys_alt, uint32_t *rows, uint32_t *rows_alt, int64_t n, int key_bytes,
                            int end_bit, void *work, int64_t work_bytes, int *result_in_alt, void *stream) {
    NBK_CHECK_ARG(n >= 0 && n < (1ll << 31), "fof_sort: row count %lld out of range", (long long)n);
    NBK_CHECK_ARG(key_bytes == 4 || key_bytes == 8, "fof_sort: keys are 4- or 8-byte integers (got %d)", key_bytes);
    NBK_CHECK_ARG(end_bit >= 1 && end_bit <= 8 * key_bytes, "fof_sort: bad key bit count %d", end_bit);
    NBK_CHECK_ARG(result_in_alt != nullptr, "fof_sort: result_in_alt is required");
    *result_in_alt = 0;
    if (n == 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    k_fof_iota<<<nbk_grid_for(n, 256, 8), 256, 0, s>>>((unsigned *)rows, n);
    NBK_LAUNCHED();
    size_t bytes = (size_t)work_bytes;
    cub::DoubleBuffer<unsigned> v((unsigned *)rows, (unsigned *)rows_alt);
    int sel;
    if (key_bytes == 8) {
        cub::DoubleBuffer<unsigned long long> k((unsigned long long *)keys, (unsigned long long *)keys_alt);
        NBK_CUDA(cub::DeviceRadixSort::SortPairs(work, bytes, k, v, (int)n, 0, end_bit, s));
        sel = k.selector;
    } else {
        cub::DoubleBuffer<unsigned> k((unsigned *)keys, (unsigned *)keys_alt);
        NBK_CUDA(cub::DeviceRadixSort::SortPairs(work, bytes, k, v, (int)n, 0, end_bit, s));
        sel = k.selector;
    }
    nbk_count_launch();
    *result_in_alt = sel;
    return NBK_OK;
}

extern "C" int nbk_fof_link(const void *sorted_pos, int pos_dtype, const uint32_t *perm, const int64_t *gid, int64_t gid_base,
                            const uint32_t *cell_start, const int64_t *cell_key, int64_t ncells, int periodic, const double *box_host,
                            const double *origin_host, const int64_t *ncell_host, double b, uint32_t *parent, int64_t *cell_min,
                            void *stream) {
    FOF_CHECK_DT(pos_dtype);
    FOF_CHECK_N(ncells);
    NBK_CHECK_ARG(gid_base >= 0, "fof_link: negative id base");
    FofGeom g;
    int rc = fof_geom(g, periodic, box_host, origin_host, ncell_host, b);
    if (rc) return rc;
    if (ncells == 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    const unsigned *cs = (const unsigned *)cell_start;
    k_fof_init<<<nbk_grid_for(ncells, 256, 8), 256, 0, s>>>(cs, ncells, (const unsigned *)perm, (const long long *)gid, gid_base,
                                                            (unsigned *)parent, (long long *)cell_min);
    NBK_LAUNCHED();
    int grid = nbk_grid_for(ncells, 128, 16);
    if (pos_dtype == NBK_F4)
        k_fof_link<float><<<grid, 128, 0, s>>>((const float *)sorted_pos, cs, (const long long *)cell_key, ncells, g, (unsigned *)parent,
                                               (const long long *)cell_min);
    else
        k_fof_link<double><<<grid, 128, 0, s>>>((const double *)sorted_pos, cs, (const long long *)cell_key, ncells, g, (unsigned *)parent,
                                                (const long long *)cell_min);
    NBK_LAUNCHED();
    k_fof_compress<<<nbk_grid_for(ncells, 256, 8), 256, 0, s>>>((unsigned *)parent, ncells);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_fof_finalize(const uint32_t *perm, const uint32_t *cell_start, int64_t ncells, const uint32_t *parent,
                                const int64_t *cell_min, uint32_t *row_root, int64_t *minid, void *stream) {
    FOF_CHECK_N(ncells);
    if (ncells == 0) return NBK_OK;
    k_fof_finalize<<<nbk_grid_for(ncells, 256, 8), 256, 0, (cudaStream_t)stream>>>(
        (const unsigned *)perm, (const unsigned *)cell_start, ncells, (const unsigned *)parent, (const long long *)cell_min,
        (unsigned *)row_root, (long long *)minid);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_fof_lower(const uint32_t *row_root, int64_t n, const int64_t *new_minid, int64_t ncells, int64_t *root_min,
                             int64_t *minid, uint64_t *changed, void *stream) {
    FOF_CHECK_N(n);
    FOF_CHECK_N(ncells);
    if (n == 0 || ncells == 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    k_fof_fill_i64<<<nbk_grid_for(ncells, 256, 8), 256, 0, s>>>((long long *)root_min, ncells, LLONG_MAX);
    NBK_LAUNCHED();
    k_fof_root_min<<<nbk_grid_for(n, 256, 8), 256, 0, s>>>((const unsigned *)row_root, n, (const long long *)new_minid, (long long *)root_min);
    NBK_LAUNCHED();
    k_fof_root_read<<<nbk_grid_for(n, 256, 8), 256, 0, s>>>((const unsigned *)row_root, n, (const long long *)root_min, (long long *)minid,
                                                            (unsigned long long *)changed);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_fof_root_counts(const uint32_t *row_root, int64_t n, uint64_t *counts, void *stream) {
    FOF_CHECK_N(n);
    if (n == 0) return NBK_OK;
    k_fof_root_counts<<<nbk_grid_for(n, 256, 8), 256, 0, (cudaStream_t)stream>>>((const unsigned *)row_root, n, (unsigned long long *)counts);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_fof_label_rows(const uint32_t *row_root, int64_t n, const int64_t *cell_label, void *labels, int label_bytes,
                                  void *stream) {
    FOF_CHECK_N(n);
    NBK_CHECK_ARG(label_bytes == 4 || label_bytes == 8, "fof_label_rows: labels are 4- or 8-byte integers (got %d)", label_bytes);
    if (n == 0) return NBK_OK;
    int grid = nbk_grid_for(n, 256, 8);
    cudaStream_t s = (cudaStream_t)stream;
    if (label_bytes == 4) k_fof_label_rows<int><<<grid, 256, 0, s>>>((const unsigned *)row_root, n, (const long long *)cell_label, (int *)labels);
    else k_fof_label_rows<long long><<<grid, 256, 0, s>>>((const unsigned *)row_root, n, (const long long *)cell_label, (long long *)labels);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_fof_segment_reduce(int op, const void *col, int col_dtype, const void *mask, int mask_dtype, const double *thresh,
                                      const double *ref, int periodic, const double *box_host, const uint32_t *order,
                                      const int64_t *chunk_first, const int64_t *chunk_label, int64_t nchunks,
                                      const int64_t *label_chunk, int64_t nlabels, double *partial, double *out, void *stream) {
    NBK_CHECK_ARG(op == NBK_FOF_RED_MIN || op == NBK_FOF_RED_MAX || op == NBK_FOF_RED_SUM, "fof_segment_reduce: bad op %d", op);
    NBK_CHECK_ARG(col_dtype == NBK_F4 || col_dtype == NBK_F8, "fof_segment_reduce: bad column dtype %d", col_dtype);
    NBK_CHECK_ARG(mask == nullptr || mask_dtype == NBK_F4 || mask_dtype == NBK_F8, "fof_segment_reduce: bad mask dtype %d", mask_dtype);
    NBK_CHECK_ARG(mask == nullptr || thresh != nullptr, "fof_segment_reduce: a mask needs per-label thresholds");
    NBK_CHECK_ARG(nchunks >= 0 && nchunks < (1ll << 31), "fof_segment_reduce: chunk count %lld out of range", (long long)nchunks);
    NBK_CHECK_ARG(nlabels >= 0 && nlabels < (1ll << 32), "fof_segment_reduce: label count %lld out of range", (long long)nlabels);
    RedArgs A;
    A.col = col; A.col_dt = col_dtype; A.mask = mask; A.mask_dt = mask_dtype; A.thresh = thresh; A.ref = ref; A.op = op;
    A.periodic = periodic ? 1 : 0;
    for (int d = 0; d < 3; d++) {
        A.box[d] = 0.0;
        if (periodic && op == NBK_FOF_RED_SUM && ref) {
            NBK_CHECK_ARG(box_host != nullptr && isfinite(box_host[d]) && box_host[d] > 0, "fof_segment_reduce: bad box");
            A.box[d] = box_host[d];
        }
    }
    if (nlabels == 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    if (nchunks > 0) {
        k_fof_reduce_chunks<<<(unsigned)nchunks, FOF_RB, 0, s>>>(A, (const unsigned *)order, (const long long *)chunk_first,
                                                                  (const long long *)chunk_label, partial);
        NBK_LAUNCHED();
    }
    k_fof_reduce_labels<<<nbk_grid_for(nlabels, 256, 8), 256, 0, s>>>(op, partial, (const long long *)label_chunk, nlabels, out);
    NBK_LAUNCHED();
    return NBK_OK;
}
