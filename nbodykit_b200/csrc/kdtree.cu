// The 8 nearest neighbours of rows of the periodic unit box (nbodykit/algorithms/kdtree.py: KDDensity; DESIGN.md 4.10)
// on a dense cell table of the cell grid of pc_cells.cuh.
//   nbk_kd_unit       : q = pos / L in the positions' dtype, then numpy's q % 1 in that dtype; a q that rounds to 1.0
//                       becomes 0.0.  Written as double.
//   nbk_kd_cell_table : the first sorted row of every cell of the grid (cells + 1 entries), from the compact cell table
//   nbk_kd_self       : per owned sorted row, the K-th smallest squared distance to every row (itself included)
//   nbk_kd_query      : per external query, the K smallest squared distances to the owned rows
//   nbk_kd_density    : d = sqrt(d2) and 1 / (d^3 V)
// Distance of unit positions a, b, all in double: dx = a_x - b_x, dx > 0.5 -> dx - 1, dx < -0.5 -> dx + 1 (the same for
// y and z), d2 = (dx^2 + dy^2) + dz^2.  The file is compiled with --fmad=false: no contraction may change d2.
#include "pc_cells.cuh"

#include <math.h>

#define KD_K 8
#define KD_B 128
#define KD_MAX_CELLS_PER_AXIS 1024

// how far a sorted row may sit outside its cell: the rounding of q * nc in the cell key, far below this
#define KD_TOL 1e-9

// numpy's float remainder by 1 (npy_divmod): fmod, + 1 when the result is negative, +0.0 for a zero result
template <typename T>
static __device__ __forceinline__ T kd_mod1(T v) {
    T m = fmod(v, (T)1);
    if (m != (T)0) {
        if (m < (T)0) m += (T)1;
    } else {
        m = (T)0;
    }
    return m == (T)1 ? (T)0 : m;
}

template <typename T>
__global__ void k_kd_unit(const T *__restrict__ pos, long long n3, double L, double *__restrict__ q) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n3; i += stride) {
        const T v = (T)((double)pos[i] / L);     // f4: f4(f8(x) / L), as numpy's in-place divide by an f8 array
        q[i] = (double)kd_mod1<T>(v);
    }
}

__global__ void k_kd_cell_table(const unsigned *__restrict__ cell_start, const long long *__restrict__ cell_key, int64_t ncells,
                                long long ntot, unsigned *__restrict__ dense) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k <= ntot; k += stride)
        dense[k] = cell_start[pc_lower_bound(cell_key, ncells, k)];
}

struct KdGrid {
    long long nc[3];
    long long lo[3], hi[3];   // the offsets -lo .. hi of an axis reach each of its cells once
    double cs[3];
};

// distance from x to the rows of unwrapped cell c of an axis (a lower bound)
static __device__ __forceinline__ double kd_direct(double x, long long c, double cs) {
    const double a = (double)c * cs - KD_TOL, b = (double)(c + 1) * cs + KD_TOL;
    return a > x ? a - x : (x > b ? x - b : 0.0);
}

// periodic distance from x (in [0, 1)) to the rows of wrapped cell w: the nearest of its three images
static __device__ __forceinline__ double kd_gap(double x, long long w, long long nc, double cs) {
    const double g0 = kd_direct(x, w, cs), g1 = kd_direct(x, w - nc, cs), g2 = kd_direct(x, w + nc, cs);
    return fmin(g0, fmin(g1, g2));
}

static __device__ __forceinline__ void kd_insert(double (&best)[KD_K], double d2) {
#pragma unroll
    for (int k = KD_K - 1; k > 0; k--) best[k] = d2 < best[k - 1] ? best[k - 1] : (d2 < best[k] ? d2 : best[k]);
    best[0] = d2 < best[0] ? d2 : best[0];
}

// The K smallest d2 from (qx, qy, qz) to the candidate rows (OWN_ONLY: those with perm < n_own), walking Chebyshev rings
// of cells around the query's cell.  A cell is skipped when its squared gap reaches the current K-th; the walk stops when
// ring R + 1 cannot beat it, when every cell has been visited, or when every candidate row has been seen.
template <bool OWN_ONLY>
static __device__ __forceinline__ void kd_walk(double qx, double qy, double qz, const double *__restrict__ spos,
                                               const unsigned *__restrict__ perm, long long n_own, long long ncand,
                                               const unsigned *__restrict__ dense, const KdGrid &g, double (&best)[KD_K],
                                               unsigned long long &cand) {
#pragma unroll
    for (int k = 0; k < KD_K; k++) best[k] = INFINITY;
    if (ncand <= 0) return;
    const double x[3] = {qx, qy, qz};
    long long ic[3];
#pragma unroll
    for (int d = 0; d < 3; d++) {
        const long long c = (long long)(x[d] * (double)g.nc[d]);
        ic[d] = c < 0 ? 0 : (c >= g.nc[d] ? g.nc[d] - 1 : c);
    }
    const long long rall = max(max(max(g.lo[0], g.hi[0]), max(g.lo[1], g.hi[1])), max(g.lo[2], g.hi[2]));
    long long seen = 0;
    for (long long R = 0;; R++) {
        const long long x0 = -min(R, g.lo[0]), x1 = min(R, g.hi[0]);
        const long long y0 = -min(R, g.lo[1]), y1 = min(R, g.hi[1]);
        const long long z0 = -min(R, g.lo[2]), z1 = min(R, g.hi[2]);
        for (long long ox = x0; ox <= x1; ox++) {
            const long long wx = pc_wrap(ic[0] + ox, g.nc[0]);
            const double gx = kd_gap(qx, wx, g.nc[0], g.cs[0]);
            const double gx2 = gx * gx;
            if (gx2 >= best[KD_K - 1]) continue;
            for (long long oy = y0; oy <= y1; oy++) {
                const long long wy = pc_wrap(ic[1] + oy, g.nc[1]);
                const double gy = kd_gap(qy, wy, g.nc[1], g.cs[1]);
                const double gxy2 = gx2 + gy * gy;
                if (gxy2 >= best[KD_K - 1]) continue;
                // the ring's cells of this column: all z offsets on its x or y faces, else only z = -R and z = R
                const bool face = ox == R || ox == -R || oy == R || oy == -R;
                const long long zstep = face ? 1 : 2 * R;
                const long long row = (wx * g.nc[1] + wy) * g.nc[2];
                for (long long oz = face ? z0 : -R; oz <= (face ? z1 : R); oz += zstep) {
                    if (oz < z0 || oz > z1) continue;
                    const long long wz = pc_wrap(ic[2] + oz, g.nc[2]);
                    const double gz = kd_gap(qz, wz, g.nc[2], g.cs[2]);
                    if (gxy2 + gz * gz >= best[KD_K - 1]) continue;
                    const long long r0 = dense[row + wz], r1 = dense[row + wz + 1];
                    for (long long j = r0; j < r1; j++) {
                        if (OWN_ONLY && (long long)perm[j] >= n_own) continue;
                        seen++;
                        double dx = qx - spos[3 * j], dy = qy - spos[3 * j + 1], dz = qz - spos[3 * j + 2];
                        if (dx > 0.5) dx -= 1.0; else if (dx < -0.5) dx += 1.0;
                        if (dy > 0.5) dy -= 1.0; else if (dy < -0.5) dy += 1.0;
                        if (dz > 0.5) dz -= 1.0; else if (dz < -0.5) dz += 1.0;
                        const double d2 = (dx * dx + dy * dy) + dz * dz;
                        if (d2 < best[KD_K - 1]) kd_insert(best, d2);
                    }
                    cand += (unsigned long long)(r1 - r0);
                }
            }
        }
        if (R >= rall || seen >= ncand) break;
        // ring R + 1: every cell of it is R + 1 cells off on some axis that still has such cells
        double lb2 = INFINITY;
#pragma unroll
        for (int d = 0; d < 3; d++) {
            if (R + 1 > max(g.lo[d], g.hi[d])) continue;
            const double a = kd_direct(x[d], ic[d] + R + 1, g.cs[d]), b = kd_direct(x[d], ic[d] - R - 1, g.cs[d]);
            const double m = fmin(a, b);
            lb2 = fmin(lb2, m * m);
        }
        if (lb2 >= best[KD_K - 1]) break;
    }
}

static __device__ __forceinline__ void kd_count(unsigned long long cand, unsigned long long *g_cand) {
    for (int o = 16; o > 0; o >>= 1) cand += __shfl_down_sync(0xffffffffu, cand, o);
    if ((threadIdx.x & 31) == 0 && cand) atomicAdd(g_cand, cand);
}

// one thread per sorted row, so that the threads of a warp walk neighbouring cells; owned rows only
__global__ void __launch_bounds__(KD_B) k_kd_self(const double *__restrict__ spos, const unsigned *__restrict__ perm, long long n,
                                                  long long n_own, const unsigned *__restrict__ dense, KdGrid g,
                                                  double *__restrict__ kth, unsigned long long *__restrict__ g_cand) {
    const long long i = (long long)blockIdx.x * KD_B + threadIdx.x;
    unsigned long long cand = 0;
    if (i < n && (long long)perm[i] < n_own) {
        double best[KD_K];
        kd_walk<false>(spos[3 * i], spos[3 * i + 1], spos[3 * i + 2], spos, perm, n_own, n, dense, g, best, cand);
        kth[perm[i]] = best[KD_K - 1];
    }
    kd_count(cand, g_cand);
}

__global__ void __launch_bounds__(KD_B) k_kd_query(const double *__restrict__ qpos, long long nq, const double *__restrict__ spos,
                                                   const unsigned *__restrict__ perm, long long n_own,
                                                   const unsigned *__restrict__ dense, KdGrid g, double *__restrict__ knn,
                                                   unsigned long long *__restrict__ g_cand) {
    const long long i = (long long)blockIdx.x * KD_B + threadIdx.x;
    unsigned long long cand = 0;
    if (i < nq) {
        double best[KD_K];
        kd_walk<true>(qpos[3 * i], qpos[3 * i + 1], qpos[3 * i + 2], spos, perm, n_own, n_own, dense, g, best, cand);
#pragma unroll
        for (int k = 0; k < KD_K; k++) knn[KD_K * i + k] = best[k];
    }
    kd_count(cand, g_cand);
}

__global__ void k_kd_density(const double *__restrict__ d2, long long n, double volume, double *__restrict__ dist,
                             double *__restrict__ density) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const double d = sqrt(d2[i]);
        dist[i] = d;
        density[i] = 1.0 / (pow(d, 3.0) * volume);
    }
}

static int kd_grid(KdGrid &g, const int64_t *ncell_host) {
    NBK_CHECK_ARG(ncell_host != nullptr, "kdtree: cell counts are required");
    for (int d = 0; d < 3; d++) {
        NBK_CHECK_ARG(ncell_host[d] >= 1 && ncell_host[d] <= KD_MAX_CELLS_PER_AXIS, "kdtree: cell count %lld on axis %d out of range",
                      (long long)ncell_host[d], d);
        g.nc[d] = ncell_host[d];
        g.lo[d] = (ncell_host[d] - 1) / 2;
        g.hi[d] = ncell_host[d] - 1 - g.lo[d];
        g.cs[d] = 1.0 / (double)ncell_host[d];
    }
    return NBK_OK;
}

extern "C" int64_t nbk_kd_k(void) { return KD_K; }

extern "C" int nbk_kd_unit(const void *pos, int pos_dtype, int64_t n, double L, double *q, void *stream) {
    NBK_CHECK_ARG(pos_dtype == NBK_F4 || pos_dtype == NBK_F8, "kdtree: positions must be float32 or float64");
    NBK_CHECK_ARG(n >= 0 && n < (1ll << 31), "kdtree: %lld rows out of range (at most 2^31 - 1)", (long long)n);
    NBK_CHECK_ARG(isfinite(L) && L > 0, "kdtree: the box side must be positive and finite (got %g)", L);
    if (n == 0) return NBK_OK;
    NBK_CHECK_ARG(pos && q, "kdtree: null device array");
    cudaStream_t s = (cudaStream_t)stream;
    const int grid = nbk_grid_for(3 * n, 256, 8);
    if (pos_dtype == NBK_F4) k_kd_unit<float><<<grid, 256, 0, s>>>((const float *)pos, 3 * n, L, q);
    else k_kd_unit<double><<<grid, 256, 0, s>>>((const double *)pos, 3 * n, L, q);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_kd_cell_table(const uint32_t *cell_start, const int64_t *cell_key, int64_t ncells, const int64_t *ncell_host,
                                 uint32_t *dense, void *stream) {
    KdGrid g;
    int rc = kd_grid(g, ncell_host);
    if (rc) return rc;
    NBK_CHECK_ARG(ncells >= 0 && ncells < (1ll << 31), "kdtree: %lld cells out of range", (long long)ncells);
    NBK_CHECK_ARG(cell_start && dense && (ncells == 0 || cell_key), "kdtree: null device array");
    const long long ntot = g.nc[0] * g.nc[1] * g.nc[2];
    cudaStream_t s = (cudaStream_t)stream;
    k_kd_cell_table<<<nbk_grid_for(ntot + 1, 256, 8), 256, 0, s>>>((const unsigned *)cell_start, (const long long *)cell_key,
                                                                  ncells, ntot, (unsigned *)dense);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_kd_self(const double *spos, const uint32_t *perm, int64_t n, int64_t n_own, const uint32_t *dense,
                           const int64_t *ncell_host, double *kth, uint64_t *candidates, void *stream) {
    NBK_CHECK_ARG(n >= 0 && n < (1ll << 31), "kdtree: %lld rows out of range (at most 2^31 - 1)", (long long)n);
    NBK_CHECK_ARG(n_own >= 0 && n_own <= n, "kdtree: %lld owned rows of %lld", (long long)n_own, (long long)n);
    KdGrid g;
    int rc = kd_grid(g, ncell_host);
    if (rc) return rc;
    if (n_own == 0) return NBK_OK;
    NBK_CHECK_ARG(spos && perm && dense && kth && candidates, "kdtree: null device array");
    cudaStream_t s = (cudaStream_t)stream;
    k_kd_self<<<(unsigned)((n + KD_B - 1) / KD_B), KD_B, 0, s>>>(spos, (const unsigned *)perm, n, n_own, (const unsigned *)dense, g,
                                                                kth, (unsigned long long *)candidates);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_kd_query(const double *qpos, int64_t nq, const double *spos, const uint32_t *perm, int64_t n, int64_t n_own,
                            const uint32_t *dense, const int64_t *ncell_host, double *knn, uint64_t *candidates, void *stream) {
    NBK_CHECK_ARG(nq >= 0 && nq < (1ll << 31), "kdtree: %lld queries out of range", (long long)nq);
    NBK_CHECK_ARG(n >= 0 && n < (1ll << 31), "kdtree: %lld rows out of range (at most 2^31 - 1)", (long long)n);
    NBK_CHECK_ARG(n_own >= 0 && n_own <= n, "kdtree: %lld owned rows of %lld", (long long)n_own, (long long)n);
    KdGrid g;
    int rc = kd_grid(g, ncell_host);
    if (rc) return rc;
    if (nq == 0) return NBK_OK;
    NBK_CHECK_ARG(qpos && knn && candidates && (n == 0 || (spos && perm && dense)), "kdtree: null device array");
    cudaStream_t s = (cudaStream_t)stream;
    if (n_own == 0) {
        k_kd_query<<<(unsigned)((nq + KD_B - 1) / KD_B), KD_B, 0, s>>>(qpos, nq, nullptr, nullptr, 0, nullptr, g, knn,
                                                                      (unsigned long long *)candidates);
    } else {
        k_kd_query<<<(unsigned)((nq + KD_B - 1) / KD_B), KD_B, 0, s>>>(qpos, nq, spos, (const unsigned *)perm, n_own,
                                                                      (const unsigned *)dense, g, knn,
                                                                      (unsigned long long *)candidates);
    }
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_kd_density(const double *d2, int64_t n, double volume, double *dist, double *density, void *stream) {
    NBK_CHECK_ARG(n >= 0, "kdtree: %lld rows out of range", (long long)n);
    NBK_CHECK_ARG(isfinite(volume) && volume > 0, "kdtree: the box volume must be positive and finite (got %g)", volume);
    if (n == 0) return NBK_OK;
    NBK_CHECK_ARG(d2 && dist && density, "kdtree: null device array");
    cudaStream_t s = (cudaStream_t)stream;
    k_kd_density<<<nbk_grid_for(n, 256, 8), 256, 0, s>>>(d2, n, volume, dist, density);
    NBK_LAUNCHED();
    return NBK_OK;
}
