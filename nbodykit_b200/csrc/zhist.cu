// The redshift histogram n(z) (nbodykit/algorithms/zhist.py: RedshiftHistogram; DESIGN.md 4.12).
//   nbk_zh_moments : count, mean, M2, min and max of the finite rows and the number of non-finite rows, in double, from
//                    per-thread Welford states fed with 4-row batches and merged by Chan's rule in a fixed order
//   nbk_zh_bin     : per row the bin i with edges[i] <= z < edges[i+1] (searchsorted(edges, z, 'right') - 1), into per-CTA
//                    shared-memory histograms flushed with global atomics, or straight into global atomics for many bins
//   nbk_zh_spline  : a cubic B-spline (t, c) at every row, as FITPACK's splev (splev.cuh: the knot interval and the
//                    de Boor-Cox recurrence of fpbspl) with its four extrapolation modes
// Redshifts and weights are float32 or float64, widened exactly to double.  Rows are 64-bit indexed.  The file is compiled
// with --fmad=false, so that the spline rounds as FITPACK's compiled without contraction does.
#include "common.cuh"
#include "splev.cuh"

#include <math.h>

#define ZH_MB 256              // threads of the moments kernels
#define ZH_PARTIALS 1056       // at most this many moment CTAs (8 per SM): their partials merge in one CTA
#define ZH_BB 512              // threads of the binning kernel
#define ZH_SMEM_BINS 4096      // bins up to this many use per-CTA shared-memory histograms (64 KB with weights)
#define ZH_SB 256              // threads of the spline kernel
#define ZH_K NBK_SPLEV_K       // spline degree

// ---------------------------------------------------------------------------------------------------------------------
// moments

struct ZhMom {
    double n, mean, m2, mn, mx, bad;
};

static __device__ __forceinline__ ZhMom zh_empty() {
    ZhMom m;
    m.n = 0.0; m.mean = 0.0; m.m2 = 0.0; m.mn = INFINITY; m.mx = -INFINITY; m.bad = 0.0;
    return m;
}

// Chan's rule: the state of the rows of a followed by those of b
static __device__ __forceinline__ void zh_merge(ZhMom &a, const ZhMom &b) {
    a.bad += b.bad;
    if (b.n == 0.0) return;
    if (a.n == 0.0) {
        const double bad = a.bad;
        a = b;
        a.bad = bad;
        return;
    }
    const double n = a.n + b.n;
    const double d = b.mean - a.mean;
    const double fb = b.n / n;
    a.mean = a.mean + d * fb;
    a.m2 = (a.m2 + b.m2) + (d * d) * (a.n * fb);
    a.n = n;
    a.mn = fmin(a.mn, b.mn);
    a.mx = fmax(a.mx, b.mx);
}

// merge the ZH_MB states of a CTA in a fixed tree; thread 0 returns the result
static __device__ __forceinline__ ZhMom zh_block_merge(ZhMom m) {
    __shared__ ZhMom sm[ZH_MB];
    sm[threadIdx.x] = m;
    __syncthreads();
    for (int s = ZH_MB / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) {
            ZhMom a = sm[threadIdx.x];
            zh_merge(a, sm[threadIdx.x + s]);
            sm[threadIdx.x] = a;
        }
        __syncthreads();
    }
    return sm[0];
}

template <typename T>
__global__ void __launch_bounds__(ZH_MB) k_zh_moments(const T *__restrict__ z, long long n, ZhMom *__restrict__ partial) {
    ZhMom m = zh_empty();
    const long long S = (long long)gridDim.x * ZH_MB;
    for (long long i0 = (long long)blockIdx.x * ZH_MB + threadIdx.x; i0 < n; i0 += 4 * S) {
        double x[4];
        bool ok[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const long long i = i0 + u * S;
            x[u] = i < n ? (double)z[i] : 0.0;
            ok[u] = i < n && isfinite(x[u]);
            if (i < n && !ok[u]) m.bad += 1.0;
        }
        // the batch as a state of its own: mean and M2 by two passes over the registers
        ZhMom b = zh_empty();
        double s = 0.0;
#pragma unroll
        for (int u = 0; u < 4; u++)
            if (ok[u]) {
                b.n += 1.0;
                s += x[u];
                b.mn = fmin(b.mn, x[u]);
                b.mx = fmax(b.mx, x[u]);
            }
        if (b.n == 0.0) continue;
        b.mean = s / b.n;
#pragma unroll
        for (int u = 0; u < 4; u++)
            if (ok[u]) {
                const double d = x[u] - b.mean;
                b.m2 += d * d;
            }
        zh_merge(m, b);
    }
    const ZhMom r = zh_block_merge(m);
    if (threadIdx.x == 0) partial[blockIdx.x] = r;
}

__global__ void __launch_bounds__(ZH_MB) k_zh_moments_final(const ZhMom *__restrict__ partial, int np, double *__restrict__ out) {
    ZhMom m = zh_empty();
    for (int k = threadIdx.x; k < np; k += ZH_MB) zh_merge(m, partial[k]);
    const ZhMom r = zh_block_merge(m);
    if (threadIdx.x == 0) {
        out[0] = r.n; out[1] = r.mean; out[2] = r.m2; out[3] = r.mn; out[4] = r.mx; out[5] = r.bad;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// binning

// the bin of x, given edges[0] <= x < edges[nb]: the largest b < nb with edges[b] <= x (edges non-decreasing)
template <bool UNIFORM>
static __device__ __forceinline__ int zh_find(double x, const double *__restrict__ edges, int nb, double inv_h) {
    if (UNIFORM) {
        // an arithmetic guess (x >= edges[0], so truncation is floor), corrected against the stored edges
        int b = (int)fmin((x - __ldg(edges)) * inv_h, (double)(nb - 1));
        while (b > 0 && x < __ldg(edges + b)) b--;
        while (b < nb - 1 && x >= __ldg(edges + b + 1)) b++;
        return b;
    }
    int lo = 0, hi = nb;                         // edges[lo] <= x < edges[hi]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(edges + mid) <= x) lo = mid;
        else hi = mid;
    }
    return lo;
}

template <bool WEIGHTED, bool UNIFORM, bool SMEM>
static __device__ __forceinline__ void zh_add(double x, double wv, const double *__restrict__ edges, int nb, double inv_h,
                                              unsigned long long *scount, double *ssum, unsigned long long *__restrict__ counts,
                                              double *__restrict__ sums) {
    const int b = zh_find<UNIFORM>(x, edges, nb, inv_h);
    if (SMEM) {
        atomicAdd(scount + b, 1ull);
        if (WEIGHTED) atomicAdd(ssum + b, wv);
    } else {
        atomicAdd(counts + b, 1ull);
        if (WEIGHTED) atomicAdd(sums + b, wv);
    }
}

template <typename T, typename W, bool WEIGHTED, bool UNIFORM, bool SMEM>
__global__ void __launch_bounds__(ZH_BB) k_zh_bin(const T *__restrict__ z, const W *__restrict__ w, long long n,
                                                  const double *__restrict__ edges, int nb, double inv_h,
                                                  unsigned long long *__restrict__ counts, double *__restrict__ sums) {
    extern __shared__ unsigned long long zh_smem[];
    unsigned long long *scount = zh_smem;
    double *ssum = reinterpret_cast<double *>(zh_smem + nb);
    if (SMEM) {
        for (int b = threadIdx.x; b < nb; b += ZH_BB) {
            scount[b] = 0ull;
            if (WEIGHTED) ssum[b] = 0.0;
        }
        __syncthreads();
    }
    const double e0 = __ldg(edges), elast = __ldg(edges + nb);
    const long long S = (long long)gridDim.x * ZH_BB;
    for (long long i0 = (long long)blockIdx.x * ZH_BB + threadIdx.x; i0 < n; i0 += 4 * S) {
        double x[4], wv[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const long long i = i0 + u * S;
            x[u] = i < n ? (double)z[i] : NAN;
            wv[u] = (WEIGHTED && i < n) ? (double)w[i] : 0.0;
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            // below the first edge, at or above the last, and NaN are not counted
            if (x[u] >= e0 && x[u] < elast) zh_add<WEIGHTED, UNIFORM, SMEM>(x[u], wv[u], edges, nb, inv_h, scount, ssum, counts, sums);
        }
    }
    if (SMEM) {
        __syncthreads();
        for (int b = threadIdx.x; b < nb; b += ZH_BB) {
            const unsigned long long c = scount[b];
            if (c) {
                atomicAdd(counts + b, c);
                if (WEIGHTED) atomicAdd(sums + b, ssum[b]);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// spline

template <typename T>
__global__ void __launch_bounds__(ZH_SB) k_zh_spline(const T *__restrict__ z, long long n, const double *__restrict__ t, int nt,
                                                     const double *__restrict__ c, int ext, double *__restrict__ out,
                                                     unsigned long long *__restrict__ outside) {
    const double tb = __ldg(t + ZH_K), te = __ldg(t + nt - ZH_K - 1);
    unsigned long long nout = 0;
    const long long S = (long long)gridDim.x * ZH_SB;
    for (long long i = (long long)blockIdx.x * ZH_SB + threadIdx.x; i < n; i += S) {
        double x = (double)z[i];
        const bool oob = x < tb || x > te;
        nout += oob;
        double v;
        if (oob && ext == 1) {
            v = 0.0;
        } else {
            if (oob && ext == 3) x = x < tb ? tb : te;
            v = nbk_splev3(x, t, nt, c);
        }
        out[i] = v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nout += __shfl_down_sync(0xffffffffu, nout, o);
    if ((threadIdx.x & 31) == 0 && nout) atomicAdd(outside, nout);
}

// ---------------------------------------------------------------------------------------------------------------------
// C ABI

extern "C" int64_t nbk_zh_smem_bins(void) { return ZH_SMEM_BINS; }

extern "C" int64_t nbk_zh_partials(void) { return ZH_PARTIALS; }

extern "C" int nbk_zh_moments(const void *z, int dtype, int64_t n, double *partial, double *out, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "zhist: redshifts must be float32 or float64");
    NBK_CHECK_ARG(n >= 0, "zhist: %lld rows out of range", (long long)n);
    NBK_CHECK_ARG((n == 0 || z) && partial && out, "zhist: null device array");
    cudaStream_t s = (cudaStream_t)stream;
    // the grid depends on n alone, so a rank's result has the same bits on every run
    const long long want = (n + 4ll * ZH_MB - 1) / (4ll * ZH_MB);
    const int grid = (int)(want < 1 ? 1 : (want > ZH_PARTIALS ? ZH_PARTIALS : want));
    ZhMom *p = reinterpret_cast<ZhMom *>(partial);
    if (dtype == NBK_F4) k_zh_moments<float><<<grid, ZH_MB, 0, s>>>((const float *)z, n, p);
    else k_zh_moments<double><<<grid, ZH_MB, 0, s>>>((const double *)z, n, p);
    NBK_LAUNCHED();
    k_zh_moments_final<<<1, ZH_MB, 0, s>>>(p, grid, out);
    NBK_LAUNCHED();
    return NBK_OK;
}

template <typename T, typename W, bool WEIGHTED, bool UNIFORM, bool SMEM>
static int zh_bin_launch(const void *z, const void *w, long long n, const double *edges, int nb, double inv_h,
                         unsigned long long *counts, double *sums, cudaStream_t s) {
    auto kern = k_zh_bin<T, W, WEIGHTED, UNIFORM, SMEM>;
    const size_t smem = SMEM ? (size_t)nb * (WEIGHTED ? 16 : 8) : 0;
    if (smem > 48 * 1024) NBK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    NBK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, ZH_BB, smem));
    if (per_sm < 1) per_sm = 1;
    const long long want = (n + 4ll * ZH_BB - 1) / (4ll * ZH_BB);
    const long long cap = (long long)per_sm * NBK_SM_COUNT;
    const int grid = (int)(want < 1 ? 1 : (want > cap ? cap : want));
    kern<<<grid, ZH_BB, smem, s>>>((const T *)z, (const W *)w, n, edges, nb, inv_h, counts, sums);
    NBK_LAUNCHED();
    return NBK_OK;
}

template <typename T, typename W, bool WEIGHTED>
static int zh_bin_paths(const void *z, const void *w, long long n, const double *edges, int nb, double inv_h,
                        unsigned long long *counts, double *sums, cudaStream_t s) {
    const bool smem = nb <= ZH_SMEM_BINS;
    if (inv_h > 0) {
        return smem ? zh_bin_launch<T, W, WEIGHTED, true, true>(z, w, n, edges, nb, inv_h, counts, sums, s)
                    : zh_bin_launch<T, W, WEIGHTED, true, false>(z, w, n, edges, nb, inv_h, counts, sums, s);
    }
    return smem ? zh_bin_launch<T, W, WEIGHTED, false, true>(z, w, n, edges, nb, inv_h, counts, sums, s)
                : zh_bin_launch<T, W, WEIGHTED, false, false>(z, w, n, edges, nb, inv_h, counts, sums, s);
}

template <typename T>
static int zh_bin_weights(const void *z, const void *w, int wdtype, long long n, const double *edges, int nb, double inv_h,
                          unsigned long long *counts, double *sums, cudaStream_t s) {
    if (!w) return zh_bin_paths<T, float, false>(z, nullptr, n, edges, nb, inv_h, counts, nullptr, s);
    if (wdtype == NBK_F4) return zh_bin_paths<T, float, true>(z, w, n, edges, nb, inv_h, counts, sums, s);
    return zh_bin_paths<T, double, true>(z, w, n, edges, nb, inv_h, counts, sums, s);
}

extern "C" int nbk_zh_bin(const void *z, int dtype, const void *w, int wdtype, int64_t n, const double *edges, int64_t nb,
                          double inv_h, uint64_t *counts, double *sums, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "zhist: redshifts must be float32 or float64");
    NBK_CHECK_ARG(!w || wdtype == NBK_F4 || wdtype == NBK_F8, "zhist: weights must be float32 or float64");
    NBK_CHECK_ARG(n >= 0, "zhist: %lld rows out of range", (long long)n);
    NBK_CHECK_ARG(nb >= 1 && nb < (1ll << 31), "zhist: %lld bins out of range (1 to 2^31 - 1)", (long long)nb);
    NBK_CHECK_ARG(isfinite(inv_h) && inv_h >= 0, "zhist: the inverse bin width must be finite and non-negative");
    if (n == 0) return NBK_OK;
    NBK_CHECK_ARG(z && edges && counts && (!w || sums), "zhist: null device array");
    cudaStream_t s = (cudaStream_t)stream;
    unsigned long long *cnt = (unsigned long long *)counts;
    if (dtype == NBK_F4) return zh_bin_weights<float>(z, w, wdtype, n, edges, (int)nb, inv_h, cnt, sums, s);
    return zh_bin_weights<double>(z, w, wdtype, n, edges, (int)nb, inv_h, cnt, sums, s);
}

extern "C" int nbk_zh_spline(const void *z, int dtype, int64_t n, const double *t, int64_t nt, const double *c, int ext,
                             double *out, uint64_t *outside, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "zhist: redshifts must be float32 or float64");
    NBK_CHECK_ARG(n >= 0, "zhist: %lld rows out of range", (long long)n);
    NBK_CHECK_ARG(nt >= 2 * (ZH_K + 1) && nt < (1ll << 31), "zhist: %lld knots out of range (at least 8)", (long long)nt);
    NBK_CHECK_ARG(ext >= 0 && ext <= 3, "zhist: extrapolation mode %d is not 0, 1, 2 or 3", ext);
    if (n == 0) return NBK_OK;
    NBK_CHECK_ARG(z && t && c && out && outside, "zhist: null device array");
    cudaStream_t s = (cudaStream_t)stream;
    const int grid = nbk_grid_for(n, ZH_SB, 8);
    if (dtype == NBK_F4)
        k_zh_spline<float><<<grid, ZH_SB, 0, s>>>((const float *)z, n, t, (int)nt, c, ext, out, (unsigned long long *)outside);
    else
        k_zh_spline<double><<<grid, ZH_SB, 0, s>>>((const double *)z, n, t, (int)nt, c, ext, out, (unsigned long long *)outside);
    NBK_LAUNCHED();
    return NBK_OK;
}
