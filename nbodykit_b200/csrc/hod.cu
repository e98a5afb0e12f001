// HOD population of halo catalogues (source/catalog/halos.py: HaloCatalog.populate; DESIGN.md 4.13).
//   nbk_hod_occupy : one thread per halo: the Zheng07 central probability and satellite mean, a Bernoulli and an exact
//                    Poisson draw (sequential inversion below a mean of 10, Hormann's PTRS above)
//   nbk_hod_occupy_smhm : the same draws for the Leauthaud11 means (the inverted Behroozi10 stellar-to-halo-mass relation,
//                    a cubic spline evaluated as FITPACK's splev), with the Heaviside assembly-bias perturbation of
//                    Hearin15 when given each halo's percentile in its mass bin
//   nbk_hod_scan   : offsets of the galaxy rows, an inclusive sum (cub) over the 2 n counts [centrals | satellites]
//   nbk_hod_emit   : one thread per galaxy: its halo by binary search over the offsets, then the NFW radius (the inverse of
//                    the truncated enclosed-mass CDF, W0 Lambert), an isotropic direction, the Jeans dispersion and
//                    Box-Muller normals
// Every uniform is a SplitMix64 hash of (seed, stream, global halo row, draw index): the catalogue does not depend on the
// number of ranks or the split of the rows.  The file is compiled with --fmad=false, so that every double operation
// rounds as the float64 NumPy restatement in oracle/hod_oracle.py does.
#include "common.cuh"
#include "splev.cuh"

#include <cub/device/device_scan.cuh>
#include <math.h>

#define HOD_OB 256            // threads of the occupation kernel
#define HOD_EB 256            // threads of the emit kernel
#define HOD_POISSON_INV 10.0  // below this mean the Poisson draw is by sequential inversion
#define HOD_INV_MAX 1000      // inversion steps at most (the CDF reaches 1 to rounding long before)
#define HOD_PTRS_MAX 100000   // PTRS attempts at most (each is accepted with probability above 0.9)

static __device__ __forceinline__ unsigned long long hod_mix(unsigned long long z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// the key of the draws of halo row h in `stream`; draw j is hod_uniform(key, j)
static __device__ __forceinline__ unsigned long long hod_key(unsigned long long seed, unsigned long long stream,
                                                             long long h) {
    return hod_mix(hod_mix(hod_mix(seed) ^ stream) ^ (unsigned long long)h);
}

// uniform in (0, 1): ((x >> 12) + 1/2) 2^-52, exact in double
static __device__ __forceinline__ double hod_uniform(unsigned long long key, long long j) {
    const unsigned long long x = hod_mix(key ^ (unsigned long long)j);
    return ((double)(x >> 12) + 0.5) * 0x1p-52;
}

// ---------------------------------------------------------------------------------------------------------------------
// occupation

// Poisson(lam) from the uniforms j = 1, 2, ... of key
static __device__ long long hod_poisson(unsigned long long key, double lam) {
    if (!(lam > 0.0)) return 0;
    if (lam < HOD_POISSON_INV) {
        const double u = hod_uniform(key, 1);
        double p = exp(-lam), s = p;
        long long x = 0;
        while (u > s && x < HOD_INV_MAX) {
            x += 1;
            p = p * (lam / (double)x);
            s = s + p;
        }
        return x;
    }
    // PTRS (Hormann 1993, "The transformed rejection method for generating Poisson random variables"), as NumPy's
    const double slam = sqrt(lam), loglam = log(lam);
    const double b = 0.931 + 2.53 * slam;
    const double a = -0.059 + 0.02483 * b;
    const double invalpha = 1.1239 + 1.1328 / (b - 3.4);
    const double vr = 0.9277 - 3.6224 / (b - 2.0);
    long long j = 1;
    for (int it = 0; it < HOD_PTRS_MAX; it++, j += 2) {
        const double U = hod_uniform(key, j) - 0.5;
        const double V = hod_uniform(key, j + 1);
        const double us = 0.5 - fabs(U);
        const double k = floor((2.0 * a / us + b) * U + lam + 0.43);
        if (us >= 0.07 && V <= vr) return (long long)k;
        if (k < 0.0 || (us < 0.013 && V > us)) continue;
        if (log(V) + log(invalpha) - log(a / (us * us) + b) <= -lam + k * loglam - lgamma(k + 1.0)) return (long long)k;
    }
    return (long long)floor(lam);   // not reached: the acceptance probability of every attempt is above 0.9
}

template <typename M>
__global__ void __launch_bounds__(HOD_OB) k_hod_occupy(const M *__restrict__ mass, long long n, long long h0, double logMmin,
                                                       double sigma_logM, double M0, double M1, double alpha, int modulate,
                                                       unsigned long long seed, long long *__restrict__ counts) {
    const long long S = (long long)gridDim.x * HOD_OB;
    for (long long i = (long long)blockIdx.x * HOD_OB + threadIdx.x; i < n; i += S) {
        const double m = (double)mass[i];
        const double p = 0.5 * (1.0 + erf((log10(m) - logMmin) / sigma_logM));
        double lam = m > M0 ? pow((m - M0) / M1, alpha) : 0.0;
        if (modulate) lam = lam * p;
        const unsigned long long key = hod_key(seed, 0, h0 + i);
        counts[i] = hod_uniform(key, 0) < p ? 1 : 0;
        counts[n + i] = hod_poisson(key, lam);
    }
}

// the Leauthaud11 / Hearin15 model: the SMHM spline (t, c) maps log10 M to the mean log10 M*, and M_sat, M_cut derive from
// the halo mass at the threshold on the host
struct HodSmhm {
    double threshold, scatter, Msat, Mcut, alphasat;
    double split, Acen, Asat;   // assembly bias: the percentile split and the strengths, in [-1, 1]
    int modulate;
};

// the Heaviside assembly-bias mean of a halo in the upper (percentile > p) or lower part of its mass bin, for the
// baseline mean nb with bounds [0, hi]: shifted by d up or by d (1 - p) / p down, so that the bin average stays nb when a
// fraction 1 - p is upper; |d| is at most what keeps both means in bounds
static __device__ __forceinline__ double hod_assembias(double nb, double A, double p, double hi, bool upper) {
    const double r = p / (1.0 - p);
    const double d = A >= 0.0 ? A * fmin(hi - nb, r * nb) : A * fmin(nb, r * (hi - nb));
    const double v = upper ? nb + d : nb - (d * (1.0 - p)) / p;
    return fmin(fmax(v, 0.0), hi);
}

template <typename M>
__global__ void __launch_bounds__(HOD_OB) k_hod_occupy_smhm(const M *__restrict__ mass, long long n, long long h0,
                                                            const double *__restrict__ t, int nt,
                                                            const double *__restrict__ c, HodSmhm q,
                                                            const double *__restrict__ pct, unsigned long long seed,
                                                            long long *__restrict__ counts) {
    const long long S = (long long)gridDim.x * HOD_OB;
    for (long long i = (long long)blockIdx.x * HOD_OB + threadIdx.x; i < n; i += S) {
        const double m = (double)mass[i];
        const double logms = nbk_splev3(log10(m), t, nt, c);
        double p = 0.5 * (1.0 - erf((q.threshold - logms) / (1.4142135623730951 * q.scatter)));
        double lam = pow(m / q.Msat, q.alphasat) * exp(-q.Mcut / m);
        if (q.modulate) lam = lam * p;
        if (pct) {
            const bool upper = pct[i] > q.split;
            p = hod_assembias(p, q.Acen, q.split, 1.0, upper);
            lam = hod_assembias(lam, q.Asat, q.split, INFINITY, upper);
        }
        const unsigned long long key = hod_key(seed, 0, h0 + i);
        counts[i] = hod_uniform(key, 0) < p ? 1 : 0;
        counts[n + i] = hod_poisson(key, lam);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// emit

// g(y) = ln(1 + y) - y / (1 + y), the NFW enclosed mass in units of 4 pi rho_s r_s^3; its series below y = 0.1
static __device__ __forceinline__ double hod_g(double y) {
    if (y < 0.1) {
        double s = 0.0;
        for (int m = 16; m >= 0; m--) s = s * (-y) + (double)(m + 1) / (double)(m + 2);
        return y * y * s;
    }
    return log1p(y) - y / (1.0 + y);
}

// y with g(y) = a (0 < a): y = -1 - 1 / W0(-exp(-1 - a)).  The starting point is the branch-point series of W0 + 1 in
// p = sqrt(2 (1 - exp(-a))) for p < 1, and the Taylor series of W0 at 0 otherwise; four Halley steps on g(y) = a, which
// has no cancellation near the branch point, finish it.
static __device__ double hod_ginv(double a) {
    const double p = sqrt(2.0 * -expm1(-a));
    double y;
    if (p < 1.0) {
        const double w = p * (1.0 + p * (-1.0 / 3.0 + p * (11.0 / 72.0 + p * (-43.0 / 540.0 + p * (769.0 / 17280.0)))));
        y = w / (1.0 - w);
    } else {
        const double z = -exp(-1.0 - a);
        const double W = z * (1.0 + z * (-1.0 + z * (1.5 + z * (-8.0 / 3.0 + z * (125.0 / 24.0)))));
        y = -1.0 - 1.0 / W;
    }
    for (int it = 0; it < 4; it++) {
        const double q = 1.0 + y;
        const double F = hod_g(y) - a;
        const double F1 = y / (q * q);
        const double F2 = (1.0 - y) / (q * q * q);
        y = y - (2.0 * F * F1) / (2.0 * F1 * F1 - F * F2);
    }
    return y;
}

// I(y) = int_y^inf g(t) / (t^3 (1 + t)^2) dt: cubic Hermite interpolation of ln I in s = ln y on the host-built table
// (tab[2k] = ln I, tab[2k + 1] = d ln I / ds at s0 + k hs, k < K); below the table I(y0) + ln(y0 / y) / 2 - 5 (y0 - y) / 3,
// above it I(y1) A(y) / A(y1) with A(y) = (4 ln y - 3) / (16 y^4), the leading terms of the series at 0 and infinity
static __device__ double hod_jeans(double y, const double *__restrict__ tab, int K, double s0, double hs) {
    const double s = log(y);
    if (s < s0) return exp(tab[0]) + 0.5 * (s0 - s) - (5.0 / 3.0) * (exp(s0) - y);
    const double s1 = s0 + (double)(K - 1) * hs;
    if (s >= s1) return exp(tab[2 * (K - 1)]) * ((4.0 * s - 3.0) / (4.0 * s1 - 3.0)) * exp(-4.0 * (s - s1));
    const double t = (s - s0) / hs;
    int k = (int)floor(t);
    if (k > K - 2) k = K - 2;
    const double f = t - (double)k;
    const double f2 = f * f, f3 = f2 * f;
    const double h00 = 2.0 * f3 - 3.0 * f2 + 1.0, h10 = f3 - 2.0 * f2 + f;
    const double h01 = -2.0 * f3 + 3.0 * f2, h11 = f3 - f2;
    const double L = h00 * tab[2 * k] + h10 * hs * tab[2 * k + 1] + h01 * tab[2 * k + 2] + h11 * hs * tab[2 * k + 3];
    return exp(L);
}

// the galaxy row r lies in entry e of the 2 n counts: offsets[e] <= r < offsets[e + 1]
static __device__ __forceinline__ long long hod_find(const long long *__restrict__ off, long long n2, long long r) {
    long long lo = 0, hi = n2;          // off[lo] <= r < off[hi]
    while (hi - lo > 1) {
        const long long mid = lo + ((hi - lo) >> 1);
        if (off[mid] <= r) lo = mid;
        else hi = mid;
    }
    return lo;
}

// x in [0, L): x - L floor(x / L) in double, then cast; a value that rounds up to L is 0
template <typename T>
static __device__ __forceinline__ T hod_wrap(double x, double L) {
    double w = x - L * floor(x / L);
    if (w >= L) w = w - L;
    if (w < 0.0) w = w + L;
    const T o = (T)w;
    return (double)o >= L ? (T)0 : o;
}

struct HodBox {
    double L[3];
};

template <typename T>
__global__ void __launch_bounds__(HOD_EB) k_hod_emit(const long long *__restrict__ off, long long n, long long ngal,
                                                     long long h0, const T *__restrict__ hpos, const T *__restrict__ hvel,
                                                     const double *__restrict__ mass, const double *__restrict__ radius,
                                                     const double *__restrict__ conc, HodBox box, double gnewton, double rsd,
                                                     const double *__restrict__ tab, int K, double s0, double hs,
                                                     unsigned long long seed, T *__restrict__ pos, T *__restrict__ vel,
                                                     T *__restrict__ voff, double *__restrict__ hcd, int *__restrict__ gal_type,
                                                     long long *__restrict__ halo_id) {
    const long long S = (long long)gridDim.x * HOD_EB;
    for (long long r = (long long)blockIdx.x * HOD_EB + threadIdx.x; r < ngal; r += S) {
        const long long e = hod_find(off, 2 * n, r);
        const bool sat = e >= n;
        const long long i = sat ? e - n : e;
        double dx[3] = {0.0, 0.0, 0.0}, dv[3] = {0.0, 0.0, 0.0}, rr = 0.0;
        if (sat) {
            const long long k = r - off[e];
            const unsigned long long key = hod_key(seed, 1, h0 + i);
            const long long j = 8 * k;
            const double c = conc[i], R = radius[i];
            const double gc = hod_g(c);
            double y = hod_ginv(hod_uniform(key, j) * gc);
            if (y > c) y = c;
            rr = (y / c) * R;
            const double mu = 2.0 * hod_uniform(key, j + 1) - 1.0;
            const double phi = 6.283185307179586 * hod_uniform(key, j + 2);
            const double st = sqrt(fmax(0.0, 1.0 - mu * mu));
            dx[0] = rr * (st * cos(phi));
            dx[1] = rr * (st * sin(phi));
            dx[2] = rr * mu;
            const double q = 1.0 + y;
            const double v2 = gnewton * mass[i] / R;
            const double sig = sqrt(v2 * (c / gc) * (y * (q * q)) * hod_jeans(y, tab, K, s0, hs));
            const double r0 = sqrt(-2.0 * log(hod_uniform(key, j + 3)));
            const double t0 = 6.283185307179586 * hod_uniform(key, j + 4);
            const double r1 = sqrt(-2.0 * log(hod_uniform(key, j + 5)));
            const double t1 = 6.283185307179586 * hod_uniform(key, j + 6);
            dv[0] = sig * (r0 * cos(t0));
            dv[1] = sig * (r0 * sin(t0));
            dv[2] = sig * (r1 * cos(t1));
        }
#pragma unroll
        for (int d = 0; d < 3; d++) {
            pos[3 * r + d] = hod_wrap<T>((double)hpos[3 * i + d] + dx[d], box.L[d]);
            const T v = (T)((double)hvel[3 * i + d] + dv[d]);
            vel[3 * r + d] = v;
            voff[3 * r + d] = (T)((double)v * rsd);
        }
        hcd[r] = rr;
        gal_type[r] = sat ? 1 : 0;
        halo_id[r] = h0 + i;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// C ABI

extern "C" int nbk_hod_occupy(const void *mass, int mdtype, int64_t n, int64_t h0, double logMmin, double sigma_logM,
                              double M0, double M1, double alpha, int modulate, uint64_t seed, int64_t *counts, void *stream) {
    NBK_CHECK_ARG(mdtype == NBK_F4 || mdtype == NBK_F8, "hod_occupy: masses must be float32 or float64");
    NBK_CHECK_ARG(n >= 0 && h0 >= 0, "hod_occupy: %lld halos from row %lld out of range", (long long)n, (long long)h0);
    NBK_CHECK_ARG(isfinite(logMmin) && isfinite(sigma_logM) && sigma_logM > 0 && M0 >= 0 && isfinite(M0) && M1 > 0 &&
                  isfinite(M1) && isfinite(alpha), "hod_occupy: invalid model parameters");
    if (n == 0) return NBK_OK;
    NBK_CHECK_ARG(mass && counts, "hod_occupy: null device array");
    cudaStream_t s = (cudaStream_t)stream;
    const int grid = nbk_grid_for(n, HOD_OB, 8);
    long long *c = (long long *)counts;
    if (mdtype == NBK_F4)
        k_hod_occupy<float><<<grid, HOD_OB, 0, s>>>((const float *)mass, n, h0, logMmin, sigma_logM, M0, M1, alpha, modulate,
                                                     seed, c);
    else
        k_hod_occupy<double><<<grid, HOD_OB, 0, s>>>((const double *)mass, n, h0, logMmin, sigma_logM, M0, M1, alpha,
                                                      modulate, seed, c);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_hod_occupy_smhm(const void *mass, int mdtype, int64_t n, int64_t h0, const double *t, int64_t nt,
                                   const double *c, double threshold, double scatter, double Msat, double Mcut,
                                   double alphasat, int modulate, const double *pct, double split, double Acen, double Asat,
                                   uint64_t seed, int64_t *counts, void *stream) {
    NBK_CHECK_ARG(mdtype == NBK_F4 || mdtype == NBK_F8, "hod_occupy_smhm: masses must be float32 or float64");
    NBK_CHECK_ARG(n >= 0 && h0 >= 0, "hod_occupy_smhm: %lld halos from row %lld out of range", (long long)n, (long long)h0);
    NBK_CHECK_ARG(nt >= 2 * (NBK_SPLEV_K + 1) && nt < (1ll << 31), "hod_occupy_smhm: %lld knots out of range (at least 8)",
                  (long long)nt);
    NBK_CHECK_ARG(isfinite(threshold) && isfinite(scatter) && scatter > 0 && isfinite(Msat) && Msat > 0 && isfinite(Mcut) &&
                  Mcut >= 0 && isfinite(alphasat), "hod_occupy_smhm: invalid model parameters");
    NBK_CHECK_ARG(!pct || (split > 0 && split < 1 && fabs(Acen) <= 1 && fabs(Asat) <= 1),
                  "hod_occupy_smhm: the split must be in (0, 1) and the assembly-bias strengths in [-1, 1]");
    if (n == 0) return NBK_OK;
    NBK_CHECK_ARG(mass && t && c && counts, "hod_occupy_smhm: null device array");
    HodSmhm q;
    q.threshold = threshold; q.scatter = scatter; q.Msat = Msat; q.Mcut = Mcut; q.alphasat = alphasat;
    q.split = split; q.Acen = Acen; q.Asat = Asat; q.modulate = modulate;
    cudaStream_t s = (cudaStream_t)stream;
    const int grid = nbk_grid_for(n, HOD_OB, 8);
    long long *cn = (long long *)counts;
    if (mdtype == NBK_F4)
        k_hod_occupy_smhm<float><<<grid, HOD_OB, 0, s>>>((const float *)mass, n, h0, t, (int)nt, c, q, pct, seed, cn);
    else
        k_hod_occupy_smhm<double><<<grid, HOD_OB, 0, s>>>((const double *)mass, n, h0, t, (int)nt, c, q, pct, seed, cn);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int64_t nbk_hod_scan_workspace(int64_t n2) {
    if (n2 < 0 || n2 >= (1ll << 31)) return -1;
    size_t bytes = 0;
    cudaError_t e = cub::DeviceScan::InclusiveSum(nullptr, bytes, (const long long *)nullptr, (long long *)nullptr, (int)n2);
    return e == cudaSuccess ? (int64_t)bytes : -1;
}

extern "C" int nbk_hod_scan(const int64_t *counts, int64_t n2, int64_t *offsets, void *work, int64_t work_bytes,
                            void *stream) {
    NBK_CHECK_ARG(n2 >= 0 && n2 < (1ll << 31), "hod_scan: %lld counts out of range", (long long)n2);
    NBK_CHECK_ARG(offsets, "hod_scan: null device array");
    cudaStream_t s = (cudaStream_t)stream;
    NBK_CUDA(cudaMemsetAsync(offsets, 0, sizeof(int64_t), s));
    if (n2 == 0) return NBK_OK;
    NBK_CHECK_ARG(counts && work, "hod_scan: null device array");
    size_t bytes = (size_t)work_bytes;
    NBK_CUDA(cub::DeviceScan::InclusiveSum(work, bytes, (const long long *)counts, (long long *)offsets + 1, (int)n2, s));
    nbk_count_launch();
    return NBK_OK;
}

template <typename T>
static int hod_emit_launch(const int64_t *off, int64_t n, int64_t ngal, int64_t h0, const void *hpos, const void *hvel,
                           const double *mass, const double *radius, const double *conc, const HodBox &box, double gnewton,
                           double rsd, const double *tab, int K, double s0, double hs, uint64_t seed, void *pos, void *vel,
                           void *voff, double *hcd, int32_t *gal_type, int64_t *halo_id, cudaStream_t s) {
    const int grid = nbk_grid_for(ngal, HOD_EB, 8);
    k_hod_emit<T><<<grid, HOD_EB, 0, s>>>((const long long *)off, n, ngal, h0, (const T *)hpos, (const T *)hvel, mass, radius,
                                          conc, box, gnewton, rsd, tab, K, s0, hs, seed, (T *)pos, (T *)vel, (T *)voff, hcd,
                                          gal_type, (long long *)halo_id);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_hod_emit(const int64_t *offsets, int64_t n, int64_t ngal, int64_t h0, const void *hpos, const void *hvel,
                            int dtype, const double *mass, const double *radius, const double *conc, const double *box_host,
                            double gnewton, double rsd, const double *table, int64_t K, double s0, double hs, uint64_t seed,
                            void *pos, void *vel, void *voff, double *hcd, int32_t *gal_type, int64_t *halo_id, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "hod_emit: positions must be float32 or float64");
    NBK_CHECK_ARG(n >= 0 && ngal >= 0 && h0 >= 0, "hod_emit: sizes out of range");
    NBK_CHECK_ARG(K >= 2 && K < (1ll << 30) && hs > 0 && isfinite(s0), "hod_emit: bad Jeans table");
    NBK_CHECK_ARG(box_host != nullptr, "hod_emit: null box");
    HodBox box;
    for (int d = 0; d < 3; d++) {
        NBK_CHECK_ARG(isfinite(box_host[d]) && box_host[d] > 0, "hod_emit: box side %d must be finite and positive", d);
        box.L[d] = box_host[d];
    }
    if (ngal == 0) return NBK_OK;
    NBK_CHECK_ARG(offsets && hpos && hvel && mass && radius && conc && table && pos && vel && voff && hcd && gal_type &&
                  halo_id, "hod_emit: null device array");
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == NBK_F4)
        return hod_emit_launch<float>(offsets, n, ngal, h0, hpos, hvel, mass, radius, conc, box, gnewton, rsd, table, (int)K,
                                      s0, hs, seed, pos, vel, voff, hcd, gal_type, halo_id, s);
    return hod_emit_launch<double>(offsets, n, ngal, h0, hpos, hvel, mass, radius, conc, box, gnewton, rsd, table, (int)K, s0,
                                   hs, seed, pos, vel, voff, hcd, gal_type, halo_id, s);
}
