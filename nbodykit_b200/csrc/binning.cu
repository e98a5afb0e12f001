// Fourier-space passes of the FFTPower path:
//   nbk_compensate        -- Field.apply(Compensate*, kind='circular')  (source/mesh/catalog.py:449-594)
//   nbk_interlace_combine -- source/mesh/catalog.py:345-347
//   nbk_power_bin         -- FFTBase._compute_3d_power (algorithms/fftpower.py:115-128) fused with
//                            project_to_basis (:507-701) / MeshSlab (meshtools.py:104-215)
//
// Built with --fmad=false: the float32 coordinate arithmetic that decides the k / mu bin of a mode
// (k_d = fl32(f32(j_d)*f32(2 pi/L_d)), k^2 = fl32(fl32(kx^2+ky^2)+kz^2), |k| = sqrt_rn, mu = div_rn)
// is part of the bit-exact contract (SURVEY B.5; pinned by nbodykit/tests/data/dataset_2d.json).
#include "common.cuh"
#include "kshell.cuh"
#include <algorithm>
#include <map>
#include <mutex>
#include <tuple>
#include <vector>
#include <math.h>
#include <stdlib.h>

#define NBK_MAX_ELL 8

// ---------------------------------------------------------------------------------------------
// compensation: v /= prod_d f(w_d), w_d = 2 pi j_d / N_d.  The factor is separable, so three 1-D
// tables of reciprocals are built once per (device, kind, N) and cached.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ double comp_factor(int kind, double w) {
    const double PI = 3.14159265358979323846;
    double s = sin(0.5 * w);
    s = s * s;
    switch (kind) {
        case NBK_COMP_CIC:
        case NBK_COMP_TSC:
        case NBK_COMP_PCS: {
            if (w == 0.0) return 1.0;
            double x = 0.5 * w;           // numpy.sinc(0.5*w/pi) = sin(0.5 w)/(0.5 w)
            double sc = sin(x) / x;
            int p = kind == NBK_COMP_CIC ? 2 : (kind == NBK_COMP_TSC ? 3 : 4);
            double r = sc;
            for (int i = 1; i < p; i++) r *= sc;
            (void)PI;
            return r;
        }
        case NBK_COMP_CIC_SHOTNOISE: return sqrt(1.0 - 2.0 / 3.0 * s);
        case NBK_COMP_TSC_SHOTNOISE: return sqrt(1.0 - s + 2.0 / 15.0 * (s * s));
        case NBK_COMP_PCS_SHOTNOISE: return sqrt(1.0 - 4.0 / 3.0 * s + 2.0 / 5.0 * (s * s) - 4.0 / 315.0 * (s * s * s));
    }
    return 1.0;
}

__global__ void k_comp_table(double *tab, int kind, int N) {
    int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < N) {
        const double TWO_PI = 6.28318530717958647692;
        double w = TWO_PI * (double)nbk_freq(j, N) / (double)N;
        tab[j] = 1.0 / comp_factor(kind, w);
    }
}

static std::mutex g_ct_mutex;
static std::map<std::tuple<int, int, int>, double *> g_ct;

static int get_comp_table(int kind, int N, cudaStream_t s, double **out) {
    int dev = 0;
    NBK_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(g_ct_mutex);
    auto key = std::make_tuple(dev, kind, N);
    auto it = g_ct.find(key);
    if (it != g_ct.end()) { *out = it->second; return NBK_OK; }
    double *p = nullptr;
    NBK_CUDA(cudaMalloc(&p, sizeof(double) * N));
    k_comp_table<<<(N + 255) / 256, 256, 0, s>>>(p, kind, N);
    NBK_LAUNCHED();
    NBK_CUDA(cudaStreamSynchronize(s));
    g_ct[key] = p;
    *out = p;
    return NBK_OK;
}

// product of two kinds' reciprocal factors along one axis (for the compensation fused into nbk_power_bin)
__global__ void k_comp_pair_table(double *tab, int kind1, int kind2, int N) {
    int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < N) {
        const double TWO_PI = 6.28318530717958647692;
        double w = TWO_PI * (double)nbk_freq(j, N) / (double)N;
        double f1 = kind1 ? 1.0 / comp_factor(kind1, w) : 1.0;
        double f2 = kind2 ? 1.0 / comp_factor(kind2, w) : 1.0;
        tab[j] = f1 * f2;
    }
}

static int get_comp_pair_table(int kind1, int kind2, int N, cudaStream_t s, double **out) {
    int dev = 0;
    NBK_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(g_ct_mutex);
    auto key = std::make_tuple(dev, 1000 + kind1 * 16 + kind2, N);
    auto it = g_ct.find(key);
    if (it != g_ct.end()) { *out = it->second; return NBK_OK; }
    double *p = nullptr;
    NBK_CUDA(cudaMalloc(&p, sizeof(double) * N));
    k_comp_pair_table<<<(N + 255) / 256, 256, 0, s>>>(p, kind1, kind2, N);
    NBK_LAUNCHED();
    NBK_CUDA(cudaStreamSynchronize(s));
    g_ct[key] = p;
    *out = p;
    return NBK_OK;
}

template <typename T>
__global__ void __launch_bounds__(256)
k_compensate(T *__restrict__ c, SlabGeom g, const double *__restrict__ t0, const double *__restrict__ t1,
             const double *__restrict__ tz) {
    // t0 / t1: tables for the first / second stored axis
    int64_t rows = (int64_t)g.count * g.D1;
    for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
        int i0 = (int)(row / g.D1), i1 = (int)(row - (int64_t)i0 * g.D1);
        double f01 = t0[g.start + i0] * t1[i1];
        T *p = c + row * (int64_t)g.Nzc * 2;
        for (int k = threadIdx.x; k < g.Nzc; k += blockDim.x) {
            double f = f01 * tz[k];
            p[2 * k] = (T)((double)p[2 * k] * f);
            p[2 * k + 1] = (T)((double)p[2 * k + 1] * f);
        }
    }
}

extern "C" int nbk_compensate(void *cplx, int dtype, int kind, const int64_t *nmesh, int transposed, int64_t start,
                              int64_t count, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "compensate: bad dtype %d", dtype);
    NBK_CHECK_ARG(kind >= NBK_COMP_CIC && kind <= NBK_COMP_PCS_SHOTNOISE, "compensate: unknown kind %d", kind);
    SlabGeom g;
    int rc = make_slab(nmesh, transposed, start, count, 1, g);
    if (rc) return rc;
    if (count == 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    double *tx, *ty, *tz;
    if ((rc = get_comp_table(kind, g.N[0], s, &tx))) return rc;
    if ((rc = get_comp_table(kind, g.N[1], s, &ty))) return rc;
    if ((rc = get_comp_table(kind, g.N[2], s, &tz))) return rc;
    int64_t rows = (int64_t)g.count * g.D1;
    int grid = (int)(rows < (int64_t)NBK_SM_COUNT * 16 ? rows : (int64_t)NBK_SM_COUNT * 16);
    int block = g.Nzc >= 256 ? 256 : 64;
    const double *t0 = g.transposed ? ty : tx, *t1 = g.transposed ? tx : ty;
    if (dtype == NBK_F4) k_compensate<float><<<grid, block, 0, s>>>((float *)cplx, g, t0, t1, tz);
    else k_compensate<double><<<grid, block, 0, s>>>((double *)cplx, g, t0, t1, tz);
    NBK_LAUNCHED();
    return NBK_OK;
}

// ---------------------------------------------------------------------------------------------
// reconstruction displacement transfer function (algorithms/fftrecon.py:213-230), kind='wavenumber':
//   out = i k_d / k^2 * in * exp(-k^2 R^2 / 2) / (bias (1 + f/bias mu^2)),  mu = k.los / |k|,  k^2 = 0 -> 1
// out of place (the density modes are reused for the three directions); f8 arithmetic, lanes along kz.
// ---------------------------------------------------------------------------------------------
struct ReconParams {
    double kf[3];      // 2 pi / L_d
    double los[3];
    double R, bias, f;
    int axis;
};

template <typename T>
__global__ void __launch_bounds__(256)
k_recon_displacement(const T *__restrict__ in, T *__restrict__ out, SlabGeom g, ReconParams q) {
    int64_t rows = (int64_t)g.count * g.D1;
    for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
        int i0 = (int)(row / g.D1), i1 = (int)(row - (int64_t)i0 * g.D1);
        int jx, jy, jz0;
        slab_freqs(g, i0, i1, 0, jx, jy, jz0);
        const double kx = (double)jx * q.kf[0], ky = (double)jy * q.kf[1];
        const double kp2 = kx * kx + ky * ky;
        const double lp = kx * q.los[0] + ky * q.los[1];
        const T *pi = in + row * (int64_t)g.Nzc * 2;
        T *po = out + row * (int64_t)g.Nzc * 2;
        for (int k = threadIdx.x; k < g.Nzc; k += blockDim.x) {
            const double kz = (double)nbk_freq(k, g.N[2]) * q.kf[2];
            double k2 = kp2 + kz * kz;
            if (k2 == 0.0) k2 = 1.0;
            const double mu = (lp + kz * q.los[2]) / sqrt(k2);
            const double frac = q.bias * (1.0 + q.f / q.bias * (mu * mu));
            const double kd = q.axis == 0 ? kx : (q.axis == 1 ? ky : kz);
            const double a = kd / k2 * (exp(-0.5 * k2 * (q.R * q.R)) / frac);
            const double re = (double)pi[2 * k], im = (double)pi[2 * k + 1];
            po[2 * k] = (T)(-a * im);          // i a (re + i im) = -a im + i a re
            po[2 * k + 1] = (T)(a * re);
        }
    }
}

extern "C" int nbk_recon_displacement(const void *in, void *out, int dtype, const int64_t *nmesh, const double *box,
                                      int transposed, int64_t start, int64_t count, int axis, double R, double bias,
                                      double f, const double *los, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "recon_displacement: bad dtype %d", dtype);
    NBK_CHECK_ARG(axis >= 0 && axis < 3, "recon_displacement: bad axis %d", axis);
    NBK_CHECK_ARG(bias != 0.0, "recon_displacement: bias must be non-zero");
    NBK_CHECK_ARG(in != nullptr && out != nullptr, "recon_displacement: null field");
    SlabGeom g;
    int rc = make_slab(nmesh, transposed, start, count, 1, g);
    if (rc) return rc;
    if (count == 0) return NBK_OK;
    ReconParams q;
    const double TWO_PI = 6.283185307179586476925286766559;
    for (int d = 0; d < 3; d++) {
        NBK_CHECK_ARG(box[d] > 0, "recon_displacement: bad BoxSize");
        q.kf[d] = TWO_PI / box[d];
        q.los[d] = los[d];
    }
    q.R = R; q.bias = bias; q.f = f; q.axis = axis;
    cudaStream_t s = (cudaStream_t)stream;
    int64_t rows = (int64_t)g.count * g.D1;
    int grid = (int)(rows < (int64_t)NBK_SM_COUNT * 16 ? rows : (int64_t)NBK_SM_COUNT * 16);
    int block = g.Nzc >= 256 ? 256 : 64;
    if (dtype == NBK_F4) k_recon_displacement<float><<<grid, block, 0, s>>>((const float *)in, (float *)out, g, q);
    else k_recon_displacement<double><<<grid, block, 0, s>>>((const double *)in, (double *)out, g, q);
    NBK_LAUNCHED();
    return NBK_OK;
}

// ---------------------------------------------------------------------------------------------
// interlacing combine: s1 = 0.5 s1 + 0.5 s2 exp(0.5 i sum_d k_d H_d), k_d H_d = 2 pi j_d / N_d
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
k_interlace(T *__restrict__ c1, const T *__restrict__ c2, SlabGeom g) {
    int64_t rows = (int64_t)g.count * g.D1;
    for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
        int i0 = (int)(row / g.D1), i1 = (int)(row - (int64_t)i0 * g.D1);
        int jx, jy, jz;
        slab_freqs(g, i0, i1, 0, jx, jy, jz);
        double base = (double)jx / (double)g.N[0] + (double)jy / (double)g.N[1];
        T *p1 = c1 + row * (int64_t)g.Nzc * 2;
        const T *p2 = c2 + row * (int64_t)g.Nzc * 2;
        for (int k = threadIdx.x; k < g.Nzc; k += blockDim.x) {
            double ph = base + (double)nbk_freq(k, g.N[2]) / (double)g.N[2];  // phase / pi
            double sn, cs;
            sincospi(ph, &sn, &cs);
            double a = p1[2 * k], b = p1[2 * k + 1], x = p2[2 * k], y = p2[2 * k + 1];
            p1[2 * k] = (T)(0.5 * a + 0.5 * (x * cs - y * sn));
            p1[2 * k + 1] = (T)(0.5 * b + 0.5 * (x * sn + y * cs));
        }
    }
}

extern "C" int nbk_interlace_combine(void *c1, const void *c2, int dtype, const int64_t *nmesh, const double *box,
                                     int transposed, int64_t start, int64_t count, void *stream) {
    (void)box;  // k_d H_d = 2 pi j_d / N_d is independent of the box size
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "interlace_combine: bad dtype %d", dtype);
    SlabGeom g;
    int rc = make_slab(nmesh, transposed, start, count, 1, g);
    if (rc) return rc;
    if (count == 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    int64_t rows = (int64_t)g.count * g.D1;
    int grid = (int)(rows < (int64_t)NBK_SM_COUNT * 16 ? rows : (int64_t)NBK_SM_COUNT * 16);
    int block = g.Nzc >= 256 ? 256 : 64;
    if (dtype == NBK_F4) k_interlace<float><<<grid, block, 0, s>>>((float *)c1, (const float *)c2, g);
    else k_interlace<double><<<grid, block, 0, s>>>((double *)c1, (const double *)c2, g);
    NBK_LAUNCHED();
    return NBK_OK;
}

// ---------------------------------------------------------------------------------------------
// power binning
// ---------------------------------------------------------------------------------------------
struct BinParams {
    SlabGeom g;
    int coord_mode;  // 4: f32 coords & mu; 8: f64 coords & mu; 48: f32 coords, f64 mu (numpy-scalar los)
    float kf32[3], los32[3];
    double kf64[3], los64[3];
    int Nx, Nmu, nb;
    int Nell;
    int ells[NBK_MAX_ELL];
    int hermitian, is_p3d, clear_zero, has_c2;
    int anti;         // the statistic obeys y(-k) = -conj y(k) (odd FKP multipoles): the fold of the mirror half flips
    int stage_edges; // the k edges fit in shared memory
    const void *c3;  // optional: the field that stands for c2 at the UNSTORED mirror mode -k (see nbk_power_bin2)
    int estride;     // 2: complex input (re, im interleaved)   1: real input (a RealField statistic, FFTCorr)
    int need_mu;     // accumulate sum(mu) per bin (musum != NULL); FFTPower mode='1d' never reads it
    int real_stat;   // the statistic is real by construction (auto power c1 conj(c1), no mirror field): no imaginary reduction
    double volume;
};

template <typename T> struct Pair2;
template <> struct Pair2<float> { typedef float2 type; };
template <> struct Pair2<double> { typedef double2 type; };

template <bool SMEM_ACC>
__device__ __forceinline__ void acc_add(double *p, double v) {
    if (v != 0.0) atomicAdd(p, v);
}

// Row sweep: one warp per (i0, i1) row of the slab, lanes strided along kz (coalesced 8/16-byte loads).
// Everything that depends on (jx, jy) only is hoisted out of the kz loop; the k bin starts from a
// uniform-spacing guess and is corrected against the exact f64 edges^2 (so it equals numpy.digitize for any
// increasing edges).  Along a row |k| is monotone in kz, so equal bins form contiguous lane runs: a
// segmented shuffle reduction leaves one shared-memory atomic per run and quantity (f64 shared atomics are
// CAS loops on sm_90a -- same-address collisions inside a warp are what make them slow, and the run
// reduction removes exactly those).  Mode counts come from the run length (no shuffle).
// LEAN: the FFTPower auto-power case (complex Hermitian field, no second / mirror field, float32 coordinates) with the
// run-time switches of the general kernel folded at compile time
template <typename T, int NELL, bool SMEM_ACC, bool SYM, bool LEAN>
__global__ void __launch_bounds__(256, (LEAN && NELL <= 3) ? 3 : 1)
k_power_bin(const T *__restrict__ c1, const T *__restrict__ c2, BinParams P, const double *__restrict__ k2edges,
            const double *__restrict__ muedges, unsigned long long *__restrict__ g_nsum, double *__restrict__ g_xsum,
            double *__restrict__ g_musum, double *__restrict__ g_ysum, double kmin, double inv_dk, int uniform,
            const double *__restrict__ ct0, const double *__restrict__ ct1, const double *__restrict__ ctz) {
    // ct0/ct1/ctz: per-axis products of the two fields' reciprocal window factors (first stored axis, second
    // stored axis, z); null when no compensation is fused
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int estride = LEAN ? 2 : P.estride;
    const int coord_mode = LEAN ? 4 : P.coord_mode;
    const bool is_p3d = LEAN ? false : (P.is_p3d != 0);
    const bool has_c2 = LEAN ? false : (P.has_c2 != 0);
    const void *c3p = LEAN ? nullptr : P.c3;
    const bool herm = LEAN ? true : (P.hermitian != 0);
    const int anti = LEAN ? 0 : P.anti;
    // shared layout: k2edges[Nx+1] | muedges[Nmu+1] | (if SMEM_ACC) xsum[nb] musum[nb] ysum[NELL][nb][2] nsum[nb](u32)
    // the k edges are staged in shared memory when they fit; with very many edges (dk = 0: one bin per distinct |k|,
    // ~N^2 of them) they stay in global memory (L2-resident) and the accumulators are global too
    const bool stage = P.stage_edges != 0;
    double *s_k2s = reinterpret_cast<double *>(smem_raw);
    double *s_mu = s_k2s + (stage ? P.Nx + 1 : 0);
    const double *s_k2 = stage ? s_k2s : k2edges;
    double *s_x = s_mu + (P.Nmu + 1);
    double *s_m = s_x + (SMEM_ACC ? P.nb : 0);
    double *s_y = s_m + (SMEM_ACC ? P.nb : 0);
    unsigned *s_n = reinterpret_cast<unsigned *>(s_y + (SMEM_ACC ? (size_t)NELL * P.nb * 2 : 0));
    if (stage) for (int i = threadIdx.x; i <= P.Nx; i += blockDim.x) s_k2s[i] = k2edges[i];
    for (int i = threadIdx.x; i <= P.Nmu; i += blockDim.x) s_mu[i] = muedges[i];
    if (SMEM_ACC) {
        int nd = P.nb * (2 + 2 * NELL);
        for (int i = threadIdx.x; i < nd; i += blockDim.x) s_x[i] = 0.0;
        for (int i = threadIdx.x; i < P.nb; i += blockDim.x) s_n[i] = 0u;
    }
    __syncthreads();

    double *a_x = SMEM_ACC ? s_x : g_xsum;
    double *a_m = SMEM_ACC ? s_m : g_musum;
    double *a_y = SMEM_ACC ? s_y : g_ysum;

    const SlabGeom &g = P.g;
    const int lane = threadIdx.x & 31;
    const int wpb = blockDim.x >> 5;
    const int nedge = P.Nx + 1;
    const int kz_iters = (g.Nzc + 31) >> 5;
    // SYM (line of sight along z): the k and mu bins, |k| and mu of a mode do not change under jx -> -jx and
    // jy -> -jy, so the (up to four) mirror rows of a canonical row (indices <= D/2) are binned together: the
    // coordinate arithmetic, the run reduction and the atomics are paid once per group, the statistic is summed
    // over the group first.  The mirror along the first stored axis is used only when the slab holds the full axis.
    const int D0 = g.transposed ? g.N[1] : g.N[0];
    const bool full0 = SYM && (g.count == D0);
    const int n0c = full0 ? (D0 / 2 + 1) : g.count;
    const int n1c = SYM ? (g.D1 / 2 + 1) : g.D1;
    const int rows = n0c * n1c;
    for (int rowc = blockIdx.x * wpb + (threadIdx.x >> 5); rowc < rows; rowc += gridDim.x * wpb) {
        int i0 = rowc / n1c, i1 = rowc - i0 * n1c;
        int jx, jy, jz0;
        slab_freqs(g, i0, i1, 0, jx, jy, jz0);
        // mirror partners (storage indices) and the multiplicity of the group
        int m0 = i0, m1 = i1;
        if (full0) { int t = (D0 - i0) % D0; if (t != i0) m0 = t; }
        if (SYM) { int t = (g.D1 - i1) % g.D1; if (t != i1) m1 = t; }
        const int mult = ((m0 != i0) ? 2 : 1) * ((m1 != i1) ? 2 : 1);
        // per-row constants, in the arithmetic the coordinate mode prescribes
        float kx32 = (float)jx * P.kf32[0], ky32 = (float)jy * P.kf32[1];
        float kp2_32 = kx32 * kx32 + ky32 * ky32;                       // (0 + kx^2) + ky^2
        float lp_32 = kx32 * P.los32[0] + ky32 * P.los32[1];            // (0 + kx l0) + ky l1
        double kx64 = (double)jx * P.kf64[0], ky64 = (double)jy * P.kf64[1];
        double kp2_64 = kx64 * kx64 + ky64 * ky64;
        double lp_64 = kx64 * P.los64[0] + ky64 * P.los64[1];
        double lp_48 = (double)kx32 * P.los64[0] + (double)ky32 * P.los64[1];
        const int64_t rowlen = (int64_t)g.Nzc * estride;
        int64_t roff[4];
        roff[0] = ((int64_t)i0 * g.D1 + i1) * rowlen;
        roff[1] = ((int64_t)i0 * g.D1 + m1) * rowlen;
        roff[2] = ((int64_t)m0 * g.D1 + i1) * rowlen;
        roff[3] = ((int64_t)m0 * g.D1 + m1) * rowlen;
        const bool use1 = (m1 != i1), use2 = (m0 != i0), use3 = use1 && use2;
        const double vol_row = ct0 ? P.volume * (ct0[g.start + i0] * ct1[i1]) : P.volume;
        // values of the (up to four) rows of the group for lane position kz; the load for round it + 1 is issued
        // before round it is binned (the sweep is bound by memory latency otherwise)
        typedef typename Pair2<T>::type V2;
        V2 cur[4], nxt[4];
        auto load_group = [&](int kz, V2 (&v)[4]) {
#pragma unroll
            for (int q = 0; q < 4; q++) {
                v[q].x = 0; v[q].y = 0;
                if (kz >= g.Nzc) continue;
                if (q == 1 && !use1) continue;
                if (q == 2 && !use2) continue;
                if (q == 3 && !use3) continue;
                if (estride == 2) v[q] = *reinterpret_cast<const V2 *>(c1 + roff[q] + 2 * kz);
                else v[q].x = c1[roff[q] + kz];
            }
        };
        load_group(lane, cur);
        for (int it = 0; it < kz_iters; it++) {
            const int kz = it * 32 + lane;
            if (it + 1 < kz_iters) load_group(kz + 32, nxt);
            int key = -1;
            double xs = 0, ms = 0, yr[NELL], yi[NELL];
            unsigned wcnt = 0;
#pragma unroll
            for (int l = 0; l < NELL; l++) { yr[l] = 0; yi[l] = 0; }
            if (kz < g.Nzc) {
                int jz = nbk_freq(kz, g.N[2]);
                double k2d, knorm, mu;
                if (coord_mode == 8) {
                    double kzv = (double)jz * P.kf64[2];
                    k2d = kp2_64 + kzv * kzv;
                    knorm = sqrt(k2d);
                    mu = (lp_64 + kzv * P.los64[2]) / knorm;
                    if (knorm == 0.0) mu = 0.0;
                } else {
                    float kzv = (float)jz * P.kf32[2];
                    float k2 = kp2_32 + kzv * kzv;
                    float kn = sqrtf(k2);   // IEEE sqrt; numpy `** 0.5` on float32 is sqrtf
                    k2d = (double)k2;
                    knorm = (double)kn;
                    if (coord_mode == 4) {
                        float m = (lp_32 + kzv * P.los32[2]) / kn;
                        mu = (kn == 0.0f) ? 0.0 : (double)m;
                    } else {
                        double m = (lp_48 + (double)kzv * P.los64[2]) / knorm;
                        mu = (kn == 0.0f) ? 0.0 : m;
                    }
                }
                // numpy.digitize(k2, edges2): number of edges <= k2
                int b = nbk_k2_bin(s_k2, nedge, k2d, knorm, kmin, inv_dk, uniform);
                int dm = 0;
                for (int i = 0; i <= P.Nmu; i++) dm += (s_mu[i] <= mu) ? 1 : 0;
                key = b * (P.Nmu + 2) + dm;
                bool nonsing = herm && (jz > 0);
                double wH = (nonsing ? 2.0 : 1.0) * (double)mult;
                wcnt = (nonsing ? 2u : 1u) * (unsigned)mult;
                xs = knorm * wH;
                ms = mu * wH;
                double yre = 0.0, yim = 0.0, zre = 0.0, zim = 0.0;     // z: c1 * conj(c3), the statistic of the mirror mode
                const bool mirror = nonsing && c3p != nullptr;
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    if (q == 1 && !use1) continue;
                    if (q == 2 && !use2) continue;
                    if (q == 3 && !use3) continue;
                    double a = (double)cur[q].x, bb = (double)cur[q].y;
                    if (is_p3d) { yre += a; yim += bb; }
                    else {
                        double c = a, d = bb;
                        if (has_c2) { const T *p2 = c2 + roff[q] + 2 * kz; c = (double)p2[0]; d = (double)p2[1]; }
                        yre += a * c + bb * d;      // c1 * conj(c2)
                        yim += bb * c - a * d;
                        if (mirror) {
                            const T *p3 = reinterpret_cast<const T *>(c3p) + roff[q] + 2 * kz;
                            const double c3r = (double)p3[0], c3i = (double)p3[1];
                            zre += a * c3r + bb * c3i;
                            zim += bb * c3r - a * c3i;
                        }
                    }
                }
                if (!is_p3d) {
                    double vol = ct0 ? vol_row * ctz[kz] : vol_row;   // V [* window compensation of both fields]
                    yre *= vol;
                    yim *= vol;
                    zre *= vol;
                    zim *= vol;
                    if (P.clear_zero && jx == 0 && jy == 0 && jz == 0) { yre = 0; yim = 0; }
                }
#pragma unroll
                for (int l = 0; l < NELL; l++) {
                    int ell = P.ells[l];
                    double f = legendre(ell, mu) * (2.0 * ell + 1.0);
                    double re = f * yre, im = f * yim;
                    if (mirror) {    // add the mirror mode from its own statistic: Leg(l)(-mu) * (+/-) conj(z)
                        const double sg = ((ell & 1) != anti) ? -1.0 : 1.0;
                        re += sg * f * zre;
                        im -= sg * f * zim;
                    } else if (nonsing) {   // add the mirror mode: Leg(l)(-mu) * (+/-) conj(y)
                        if ((ell & 1) != anti) { re = 0.0; im *= 2.0; }
                        else { re *= 2.0; im = 0.0; }
                    }
                    yr[l] = re;
                    yi[l] = im;
                }
            }
            // ---- equal-key runs of lanes -> one atomic per run
            int prev = __shfl_up_sync(0xffffffffu, key, 1);
            bool head = (lane == 0) || (prev != key);
            unsigned heads = __ballot_sync(0xffffffffu, head);
            // count: all members of a run share wcnt except the kz = 0 / Nyquist planes -> reduce it as an int
            if (heads == 0xffffffffu) {
                // every lane is its own run: nothing to combine
            } else if (heads == 1u) {
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    wcnt += __shfl_xor_sync(0xffffffffu, wcnt, o);
                    xs += __shfl_xor_sync(0xffffffffu, xs, o);
                    if (P.need_mu) ms += __shfl_xor_sync(0xffffffffu, ms, o);
#pragma unroll
                    for (int l = 0; l < NELL; l++) {
                        yr[l] += __shfl_xor_sync(0xffffffffu, yr[l], o);
                        if (!P.real_stat) yi[l] += __shfl_xor_sync(0xffffffffu, yi[l], o);
                    }
                }
            } else {
                // longest run bounds the number of doubling steps needed
                unsigned hm = heads;
                int seg = __popc(hm & (0xffffffffu >> (31 - lane)));
                int maxrun = 1;
                {   // run length of my segment = distance between my head and the next head
                    unsigned above = hm & ~((2u << lane) - 1u);          // heads strictly above me
                    int next = above ? (__ffs(above) - 1) : 32;
                    unsigned below = hm & ((2u << lane) - 1u);           // heads at or below me
                    int mine = 31 - __clz(below);
                    maxrun = next - mine;
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) maxrun = max(maxrun, __shfl_xor_sync(0xffffffffu, maxrun, o));
                for (int o = 1; o < maxrun; o <<= 1) {
                    int so = __shfl_down_sync(0xffffffffu, seg, o);
                    bool take = (lane + o < 32) && (so == seg);
                    unsigned c_o = __shfl_down_sync(0xffffffffu, wcnt, o);
                    double x_o = __shfl_down_sync(0xffffffffu, xs, o);
                    if (take) { wcnt += c_o; xs += x_o; }
                    if (P.need_mu) {
                        double m_o = __shfl_down_sync(0xffffffffu, ms, o);
                        if (take) ms += m_o;
                    }
#pragma unroll
                    for (int l = 0; l < NELL; l++) {
                        double r_o = __shfl_down_sync(0xffffffffu, yr[l], o);
                        if (take) yr[l] += r_o;
                        if (!P.real_stat) {
                            double i_o = __shfl_down_sync(0xffffffffu, yi[l], o);
                            if (take) yi[l] += i_o;
                        }
                    }
                }
            }
            if (head && key >= 0) {
                if (SMEM_ACC) atomicAdd(&s_n[key], wcnt);
                else atomicAdd(&g_nsum[key], (unsigned long long)wcnt);
                acc_add<SMEM_ACC>(&a_x[key], xs);
                if (P.need_mu) acc_add<SMEM_ACC>(&a_m[key], ms);
#pragma unroll
                for (int l = 0; l < NELL; l++) {
                    acc_add<SMEM_ACC>(&a_y[((size_t)l * P.nb + key) * 2], yr[l]);
                    acc_add<SMEM_ACC>(&a_y[((size_t)l * P.nb + key) * 2 + 1], yi[l]);
                }
            }
#pragma unroll
            for (int q = 0; q < 4; q++) cur[q] = nxt[q];
        }
    }
    if (SMEM_ACC) {
        __syncthreads();
        for (int i = threadIdx.x; i < P.nb; i += blockDim.x) {
            unsigned c = s_n[i];
            if (c) atomicAdd(&g_nsum[i], (unsigned long long)c);
            if (s_x[i] != 0.0) atomicAdd(&g_xsum[i], s_x[i]);
            if (P.need_mu && s_m[i] != 0.0) atomicAdd(&g_musum[i], s_m[i]);
        }
        for (int i = threadIdx.x; i < NELL * P.nb * 2; i += blockDim.x)
            if (s_y[i] != 0.0) atomicAdd(&g_ysum[i], s_y[i]);
    }
}

// device copies of the edge arrays, cached per (device, content)
struct EdgeCache {
    std::vector<double> host;
    double *dev = nullptr;
};
static std::mutex g_edge_mutex;
static std::map<int, std::vector<EdgeCache>> g_edges;

static int get_edges(const double *host, int n, cudaStream_t s, double **out) {
    int dev = 0;
    NBK_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(g_edge_mutex);
    auto &vec = g_edges[dev];
    // LRU: a hit moves the entry to the back, a miss on a full cache evicts the FRONT entry only -- so an array handed
    // out earlier in the same nbk_* call (the k edges, when the mu edges miss) is never the one freed.  cudaFree
    // synchronises the device, so kernels still reading the evicted array have finished.
    for (size_t i = 0; i < vec.size(); i++) {
        if ((int)vec[i].host.size() == n && memcmp(vec[i].host.data(), host, sizeof(double) * n) == 0) {
            if (i + 1 != vec.size()) std::rotate(vec.begin() + i, vec.begin() + i + 1, vec.end());
            *out = vec.back().dev;
            return NBK_OK;
        }
    }
    if (vec.size() >= 64) {  // bounded cache
        cudaFree(vec.front().dev);
        vec.erase(vec.begin());
    }
    EdgeCache c;
    c.host.assign(host, host + n);
    NBK_CUDA(cudaMalloc(&c.dev, sizeof(double) * n));
    NBK_CUDA(cudaMemcpyAsync(c.dev, c.host.data(), sizeof(double) * n, cudaMemcpyHostToDevice, s));
    NBK_CUDA(cudaStreamSynchronize(s));
    vec.push_back(c);
    *out = vec.back().dev;
    return NBK_OK;
}

template <typename T, int NELL>
static int launch_bin(const void *c1, const void *c2, const BinParams &P, const double *d_k2, const double *d_mu,
                      int64_t *nsum, double *xsum, double *musum, double *ysum, double kmin, double inv_dk, int uniform,
                      const double *ct0, const double *ct1, const double *ctz, cudaStream_t s) {
    size_t edge_bytes = sizeof(double) * (P.Nx + 1 + P.Nmu + 1);
    size_t acc_bytes = (size_t)P.nb * (sizeof(double) * (2 + 2 * NELL) + sizeof(unsigned));
    bool smem_acc = edge_bytes + acc_bytes <= 200 * 1024;
    const bool stage = edge_bytes <= 200 * 1024 && getenv("NBK_BIN_EDGES_GLOBAL") == nullptr;   // (env: force the global path)
    if (!stage) edge_bytes = sizeof(double) * (P.Nmu + 1);      // k edges read from global memory
    size_t smem = edge_bytes + (smem_acc ? acc_bytes : 0);
    NBK_CHECK_ARG(smem <= 227 * 1024, "power_bin: too many mu edges for shared memory");
    BinParams Pk = P;
    Pk.stage_edges = stage ? 1 : 0;
    int64_t rows = (int64_t)P.g.count * P.g.D1;
    int per_sm = (int)((220 * 1024) / (smem + 1024));
    if (per_sm > 8) per_sm = 8;
    if (per_sm < 1) per_sm = 1;
    int64_t want = (rows + 7) / 8;
    int grid = (int)(want < (int64_t)NBK_SM_COUNT * per_sm ? want : (int64_t)NBK_SM_COUNT * per_sm);
    if (grid < 1) grid = 1;
    // mirror symmetry is usable when mu does not depend on kx, ky (line of sight along z)
    const bool sym = (P.los64[0] == 0.0 && P.los64[1] == 0.0);
#define LAUNCH_BIN(ACC, SYMV, LEANV)                                                                                        \
    do {                                                                                                             \
        NBK_CUDA(cudaFuncSetAttribute(k_power_bin<T, NELL, ACC, SYMV, LEANV>, cudaFuncAttributeMaxDynamicSharedMemorySize,   \
                                      (int)smem));                                                                   \
        int occ = 1;   /* persistent row loop: exactly one wave of resident CTAs */                                   \
        NBK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_power_bin<T, NELL, ACC, SYMV, LEANV>, 256, smem));    \
        if (occ < 1) occ = 1;                                                                                        \
        if ((int64_t)grid > (int64_t)NBK_SM_COUNT * occ) grid = NBK_SM_COUNT * occ;                                   \
        k_power_bin<T, NELL, ACC, SYMV, LEANV><<<grid, 256, smem, s>>>((const T *)c1, (const T *)c2, Pk, d_k2, d_mu,         \
                                                                (unsigned long long *)nsum, xsum, musum, ysum, kmin, \
                                                                inv_dk, uniform, ct0, ct1, ctz);                      \
    } while (0)
    const bool lean = smem_acc && !P.is_p3d && !P.has_c2 && P.c3 == nullptr && P.estride == 2 && P.coord_mode == 4 &&
                      P.hermitian == 1 && P.anti == 0;
    if (lean) { if (sym) LAUNCH_BIN(true, true, true); else LAUNCH_BIN(true, false, true); }
    else if (smem_acc) { if (sym) LAUNCH_BIN(true, true, false); else LAUNCH_BIN(true, false, false); }
    else { if (sym) LAUNCH_BIN(false, true, false); else LAUNCH_BIN(false, false, false); }
#undef LAUNCH_BIN
    NBK_LAUNCHED();
    return NBK_OK;
}

template <typename T>
static int launch_bin_ell(const void *c1, const void *c2, const BinParams &P, const double *d_k2, const double *d_mu,
                          int64_t *nsum, double *xsum, double *musum, double *ysum, double kmin, double inv_dk,
                          int uniform, const double *ct0, const double *ct1, const double *ctz, cudaStream_t s) {
    switch (P.Nell) {
        case 1: return launch_bin<T, 1>(c1, c2, P, d_k2, d_mu, nsum, xsum, musum, ysum, kmin, inv_dk, uniform, ct0, ct1, ctz, s);
        case 2: return launch_bin<T, 2>(c1, c2, P, d_k2, d_mu, nsum, xsum, musum, ysum, kmin, inv_dk, uniform, ct0, ct1, ctz, s);
        case 3: return launch_bin<T, 3>(c1, c2, P, d_k2, d_mu, nsum, xsum, musum, ysum, kmin, inv_dk, uniform, ct0, ct1, ctz, s);
        case 4: return launch_bin<T, 4>(c1, c2, P, d_k2, d_mu, nsum, xsum, musum, ysum, kmin, inv_dk, uniform, ct0, ct1, ctz, s);
        case 5: return launch_bin<T, 5>(c1, c2, P, d_k2, d_mu, nsum, xsum, musum, ysum, kmin, inv_dk, uniform, ct0, ct1, ctz, s);
        case 6: return launch_bin<T, 6>(c1, c2, P, d_k2, d_mu, nsum, xsum, musum, ysum, kmin, inv_dk, uniform, ct0, ct1, ctz, s);
        case 7: return launch_bin<T, 7>(c1, c2, P, d_k2, d_mu, nsum, xsum, musum, ysum, kmin, inv_dk, uniform, ct0, ct1, ctz, s);
        case 8: return launch_bin<T, 8>(c1, c2, P, d_k2, d_mu, nsum, xsum, musum, ysum, kmin, inv_dk, uniform, ct0, ct1, ctz, s);
    }
    nbk_set_error("power_bin: Nell=%d unsupported (1..%d)", P.Nell, NBK_MAX_ELL);
    return NBK_ERR_UNSUPPORTED;
}

static int power_bin_impl(const void *c1, const void *c2, const void *c3, int dtype, int is_p3d, double volume, int clear_zero,
                          const int64_t *nmesh, const double *box, int transposed, int64_t start, int64_t count,
                          int coord_dtype, const double *k2edges, int Nx, const double *muedges, int Nmu,
                          const double *los, const int *ells, int Nell, int hermitian, int comp1, int comp2,
                          int real_input, const double *coord_unit, int64_t *nsum, double *xsum, double *musum,
                          double *ysum, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "power_bin: bad dtype %d", dtype);
    NBK_CHECK_ARG(coord_dtype == 4 || coord_dtype == 8 || coord_dtype == 48, "power_bin: bad coord_dtype %d", coord_dtype);
    NBK_CHECK_ARG(Nx >= 0 && Nmu >= 1, "power_bin: need Nx >= 0 and Nmu >= 1");
    NBK_CHECK_ARG((int64_t)nmesh[0] * nmesh[1] < (1ll << 31), "power_bin: too many rows");
    NBK_CHECK_ARG(Nell >= 1 && Nell <= NBK_MAX_ELL && ells[0] == 0, "power_bin: ells must start with 0, 1 <= Nell <= %d", NBK_MAX_ELL);
    BinParams P;
    int rc = make_slab(nmesh, transposed, start, count, hermitian, P.g);
    if (rc) return rc;
    if (count == 0) return NBK_OK;
    P.coord_mode = coord_dtype;
    const double TWO_PI = 6.283185307179586476925286766559;
    for (int d = 0; d < 3; d++) {
        NBK_CHECK_ARG(box[d] > 0, "power_bin: bad BoxSize");
        P.kf64[d] = coord_unit ? coord_unit[d] : TWO_PI / box[d];
        P.kf32[d] = (float)P.kf64[d];
        P.los64[d] = los[d];
        P.los32[d] = (float)los[d];
    }
    P.Nx = Nx; P.Nmu = Nmu; P.nb = (Nx + 2) * (Nmu + 2);
    P.Nell = Nell;
    for (int l = 0; l < NBK_MAX_ELL; l++) P.ells[l] = l < Nell ? ells[l] : 0;
    for (int l = 0; l < Nell; l++) NBK_CHECK_ARG(ells[l] >= 0 && ells[l] <= 64, "power_bin: bad multipole %d", ells[l]);
    P.hermitian = hermitian ? 1 : 0;
    P.anti = hermitian == 2 ? 1 : 0;
    P.is_p3d = is_p3d ? 1 : 0;
    P.estride = real_input ? 1 : 2;
    NBK_CHECK_ARG(!real_input || (is_p3d && !hermitian), "power_bin: a real input must be a full (non-Hermitian) 3-D statistic");
    P.clear_zero = clear_zero ? 1 : 0;
    P.has_c2 = (c2 != nullptr && c2 != c1) ? 1 : 0;
    P.c3 = (c3 != nullptr && hermitian && !is_p3d && !real_input) ? c3 : nullptr;
    P.volume = volume;
    P.need_mu = musum != nullptr ? 1 : 0;
    P.real_stat = (!is_p3d && !real_input && !P.has_c2 && P.c3 == nullptr) ? 1 : 0;    // |c1|^2 V: the imaginary part is exactly 0
    cudaStream_t s = (cudaStream_t)stream;
    double *d_k2, *d_mu;
    if ((rc = get_edges(k2edges, Nx + 1, s, &d_k2))) return rc;
    if ((rc = get_edges(muedges, Nmu + 1, s, &d_mu))) return rc;
    // fused window compensation: per-axis products of the two fields' reciprocal factors
    const double *ct0 = nullptr, *ct1 = nullptr, *ctz = nullptr;
    if (!is_p3d && (comp1 != NBK_COMP_NONE || comp2 != NBK_COMP_NONE)) {
        NBK_CHECK_ARG(comp1 >= 0 && comp1 <= NBK_COMP_PCS_SHOTNOISE && comp2 >= 0 && comp2 <= NBK_COMP_PCS_SHOTNOISE,
                      "power_bin: unknown compensation kind");
        if (c2 == nullptr || c2 == c1) comp2 = comp1;
        double *t[3];
        for (int d = 0; d < 3; d++)
            if ((rc = get_comp_pair_table(comp1, comp2, P.g.N[d], s, &t[d]))) return rc;
        ct0 = P.g.transposed ? t[1] : t[0];
        ct1 = P.g.transposed ? t[0] : t[1];
        ctz = t[2];
    }
    // are the k edges uniformly spaced (numpy.arange)?  then bins start from a closed-form guess
    double kmin, inv_dk;
    const int uniform = nbk_k2_uniform(k2edges, Nx, &kmin, &inv_dk);
    if (dtype == NBK_F4) return launch_bin_ell<float>(c1, c2, P, d_k2, d_mu, nsum, xsum, musum, ysum, kmin, inv_dk, uniform, ct0, ct1, ctz, s);
    return launch_bin_ell<double>(c1, c2, P, d_k2, d_mu, nsum, xsum, musum, ysum, kmin, inv_dk, uniform, ct0, ct1, ctz, s);
}

extern "C" int nbk_power_bin(const void *c1, const void *c2, int dtype, int is_p3d, double volume, int clear_zero,
                             const int64_t *nmesh, const double *box, int transposed, int64_t start, int64_t count,
                             int coord_dtype, const double *k2edges, int Nx, const double *muedges, int Nmu,
                             const double *los, const int *ells, int Nell, int hermitian, int comp1, int comp2,
                             int real_input, const double *coord_unit, int64_t *nsum, double *xsum, double *musum,
                             double *ysum, void *stream) {
    return power_bin_impl(c1, c2, nullptr, dtype, is_p3d, volume, clear_zero, nmesh, box, transposed, start, count, coord_dtype,
                          k2edges, Nx, muedges, Nmu, los, ells, Nell, hermitian, comp1, comp2, real_input, coord_unit, nsum,
                          xsum, musum, ysum, stream);
}

// FFTPower mode '1d' auto power of a single-rank Hermitian-compressed field that still lacks its x pass: the x pass
// (scaled by extra_scale / prod(N)) fused with nbk_power_bin's binning, float32 coordinates (coord_dtype 4), poles [0],
// zero mode cleared.  *fused = 0 when the shape or the binning does not take the fused kernel (f4, line of sight not
// along z, mu edges other than {-1, 1}, Nx not in {256, 512, 1024}, too many k bins for shared memory): nothing ran and the
// caller finishes the transform and bins as usual.
extern "C" int nbk_fft_x_power_bin(void *cplx, int dtype, const int64_t *nmesh, const double *box, double extra_scale,
                                   double volume, const double *k2edges, int Nx, const double *muedges, int Nmu,
                                   const double *los, int comp, int64_t *nsum, double *xsum, double *ysum, int *fused,
                                   void *stream) {
    NBK_CHECK_ARG(fused != nullptr, "fft_x_power_bin: null result flag");
    *fused = 0;
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "fft_x_power_bin: bad dtype %d", dtype);
    NBK_CHECK_ARG(Nx >= 0 && Nmu >= 1, "fft_x_power_bin: need Nx >= 0 and Nmu >= 1");
    NBK_CHECK_ARG(comp >= 0 && comp <= NBK_COMP_PCS_SHOTNOISE, "fft_x_power_bin: unknown compensation kind %d", comp);
    SlabGeom g;
    int rc = make_slab(nmesh, 0, 0, nmesh[0], 1, g);
    if (rc) return rc;
    if (Nmu != 1 || muedges[0] != -1.0 || muedges[1] != 1.0 || los[0] != 0.0 || los[1] != 0.0) return NBK_OK;
    XBinArgs a;
    const double TWO_PI = 6.283185307179586476925286766559;
    for (int d = 0; d < 3; d++) {
        NBK_CHECK_ARG(box[d] > 0, "fft_x_power_bin: bad BoxSize");
        a.N[d] = g.N[d];
        a.kf32[d] = (float)(TWO_PI / box[d]);
    }
    a.Nzc = g.Nzc;
    a.losz32 = (float)los[2];
    a.volume = volume;
    a.nedge = Nx + 1;
    cudaStream_t s = (cudaStream_t)stream;
    double *d_k2;
    if ((rc = get_edges(k2edges, Nx + 1, s, &d_k2))) return rc;
    a.k2edges = d_k2;
    a.uniform = nbk_k2_uniform(k2edges, Nx, &a.kmin, &a.inv_dk);
    a.ct0 = a.ct1 = a.ctz = nullptr;
    if (comp != NBK_COMP_NONE) {
        double *t[3];
        for (int d = 0; d < 3; d++)
            if ((rc = get_comp_pair_table(comp, comp, g.N[d], s, &t[d]))) return rc;
        a.ct0 = t[0];
        a.ct1 = t[1];
        a.ctz = t[2];
    }
    a.nsum = (unsigned long long *)nsum;
    a.xsum = xsum;
    a.ysum = ysum;
    const double scale = extra_scale / ((double)g.N[0] * (double)g.N[1] * (double)g.N[2]);   // as nbk_r2c
    bool done = false;
    if ((rc = fft_x_bin_launch(cplx, dtype, scale, a, s, &done))) return rc;
    *fused = done ? 1 : 0;
    return NBK_OK;
}

extern "C" int nbk_power_bin2(const void *c1, const void *c2, const void *c2_mirror, int dtype, int is_p3d, double volume,
                              int clear_zero, const int64_t *nmesh, const double *box, int transposed, int64_t start,
                              int64_t count, int coord_dtype, const double *k2edges, int Nx, const double *muedges, int Nmu,
                              const double *los, const int *ells, int Nell, int hermitian, int comp1, int comp2,
                              int real_input, const double *coord_unit, int64_t *nsum, double *xsum, double *musum,
                              double *ysum, void *stream) {
    return power_bin_impl(c1, c2, c2_mirror, dtype, is_p3d, volume, clear_zero, nmesh, box, transposed, start, count,
                          coord_dtype, k2edges, Nx, muedges, Nmu, los, ells, Nell, hermitian, comp1, comp2, real_input,
                          coord_unit, nsum, xsum, musum, ysum, stream);
}
