// Error state, launch accounting and the elementwise/reduction helpers behind
// RealField/ComplexField in-place arithmetic.
#include "common.cuh"
#include <atomic>
#include <string.h>

static thread_local char g_err[1024] = "";
static std::atomic<int64_t> g_launches{0};

void nbk_set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
void nbk_count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

extern "C" int nbk_version(void) { return 104; }
extern "C" const char *nbk_last_error(void) { return g_err; }
extern "C" int64_t nbk_launch_count(void) { return g_launches.load(); }

// ---------------------------------------------------------------------------------------------
// streaming elementwise kernels: 128-bit accesses on the aligned body, scalar tail.
// ---------------------------------------------------------------------------------------------
template <typename T> struct Vec16;
template <> struct Vec16<float> { typedef float4 type; enum { N = 4 }; };
template <> struct Vec16<double> { typedef double2 type; enum { N = 2 }; };

template <typename T, int OP>  // OP 0: fill, 1: scale
__global__ void __launch_bounds__(256) k_unary(T *__restrict__ x, int64_t n, T a) {
    typedef typename Vec16<T>::type V;
    const int VN = Vec16<T>::N;
    int64_t nv = n / VN;
    V *xv = reinterpret_cast<V *>(x);
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += stride) {
        V v;
        T *e = reinterpret_cast<T *>(&v);
        if (OP == 1) {
            v = xv[i];
#pragma unroll
            for (int k = 0; k < VN; k++) e[k] *= a;
        } else {
#pragma unroll
            for (int k = 0; k < VN; k++) e[k] = a;
        }
        xv[i] = v;
    }
    for (int64_t i = nv * VN + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        x[i] = (OP == 1) ? x[i] * a : a;
}

template <typename T>
__global__ void __launch_bounds__(256) k_axpy(T *__restrict__ y, const T *__restrict__ x, int64_t n, T a) {
    typedef typename Vec16<T>::type V;
    const int VN = Vec16<T>::N;
    int64_t nv = n / VN;
    V *yv = reinterpret_cast<V *>(y);
    const V *xv = reinterpret_cast<const V *>(x);
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += stride) {
        V vy = yv[i], vx = xv[i];
        T *ey = reinterpret_cast<T *>(&vy);
        const T *ex = reinterpret_cast<const T *>(&vx);
#pragma unroll
        for (int k = 0; k < VN; k++) ey[k] += a * ex[k];
        yv[i] = vy;
    }
    for (int64_t i = nv * VN + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        y[i] += a * x[i];
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// out[0] += sum x ; if SQ: out[1] += sum x^2.  f8 accumulation, one REDG.F64 per CTA.
template <typename T, bool SQ>
__global__ void __launch_bounds__(256) k_sum(const T *__restrict__ x, int64_t n, double *__restrict__ out) {
    double s = 0, s2 = 0;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        double v = (double)x[i];
        s += v;
        if (SQ) s2 += v * v;
    }
    __shared__ double sh[2][8];
    s = warp_sum(s);
    if (SQ) s2 = warp_sum(s2);
    int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) { sh[0][w] = s; sh[1][w] = s2; }
    __syncthreads();
    if (w == 0) {
        s = (l < 8) ? sh[0][l] : 0.0;
        s2 = (l < 8) ? sh[1][l] : 0.0;
        s = warp_sum(s);
        if (SQ) s2 = warp_sum(s2);
        if (l == 0) {
            atomicAdd(&out[0], s);
            if (SQ) atomicAdd(&out[1], s2);
        }
    }
}

// out = c1 * conj(c2) * scale, element 0 optionally cleared (FFTBase._compute_3d_power, fftpower.py:115-128;
// materialised only for FFTCorr, which transforms the 3-D power back to configuration space)
template <typename T>
__global__ void __launch_bounds__(256)
k_cross_power(const T *__restrict__ c1, const T *__restrict__ c2, T *__restrict__ out, int64_t n, T scale, int clear_first) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        T a = c1[2 * i], b = c1[2 * i + 1], c = c2[2 * i], d = c2[2 * i + 1];
        T re = (a * c + b * d) * scale, im = (b * c - a * d) * scale;
        if (clear_first && i == 0) { re = 0; im = 0; }
        out[2 * i] = re;
        out[2 * i + 1] = im;
    }
}

extern "C" int nbk_cross_power(const void *c1, const void *c2, void *out, int dtype, int64_t n_complex, double scale,
                               int clear_first, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "nbk_cross_power: bad dtype %d", dtype);
    if (n_complex <= 0) return NBK_OK;
    if (c2 == nullptr) c2 = c1;
    cudaStream_t s = (cudaStream_t)stream;
    int g = nbk_grid_for(n_complex, 256, 8);
    if (dtype == NBK_F4) k_cross_power<float><<<g, 256, 0, s>>>((const float *)c1, (const float *)c2, (float *)out, n_complex, (float)scale, clear_first);
    else k_cross_power<double><<<g, 256, 0, s>>>((const double *)c1, (const double *)c2, (double *)out, n_complex, scale, clear_first);
    NBK_LAUNCHED();
    return NBK_OK;
}

static bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int nbk_fill(void *x, int dtype, int64_t n, double value, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "nbk_fill: bad dtype %d", dtype);
    NBK_CHECK_ARG(aligned16(x), "nbk_fill: pointer must be 16-byte aligned");
    if (n <= 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    int g = nbk_grid_for(n / 4 + 1, 256, 8);
    if (dtype == NBK_F4) k_unary<float, 0><<<g, 256, 0, s>>>((float *)x, n, (float)value);
    else k_unary<double, 0><<<g, 256, 0, s>>>((double *)x, n, value);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_scale(void *x, int dtype, int64_t n, double a, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "nbk_scale: bad dtype %d", dtype);
    NBK_CHECK_ARG(aligned16(x), "nbk_scale: pointer must be 16-byte aligned");
    if (n <= 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    int g = nbk_grid_for(n / 4 + 1, 256, 8);
    if (dtype == NBK_F4) k_unary<float, 1><<<g, 256, 0, s>>>((float *)x, n, (float)a);
    else k_unary<double, 1><<<g, 256, 0, s>>>((double *)x, n, a);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_axpy(void *y, const void *x, int dtype, int64_t n, double a, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "nbk_axpy: bad dtype %d", dtype);
    NBK_CHECK_ARG(aligned16(x) && aligned16(y), "nbk_axpy: pointers must be 16-byte aligned");
    if (n <= 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    int g = nbk_grid_for(n / 4 + 1, 256, 8);
    if (dtype == NBK_F4) k_axpy<float><<<g, 256, 0, s>>>((float *)y, (const float *)x, n, (float)a);
    else k_axpy<double><<<g, 256, 0, s>>>((double *)y, (const double *)x, n, a);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_sum(const void *x, int dtype, int64_t n, double *out1, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "nbk_sum: bad dtype %d", dtype);
    if (n <= 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    int g = nbk_grid_for(n, 256, 4);
    if (dtype == NBK_F4) k_sum<float, false><<<g, 256, 0, s>>>((const float *)x, n, out1);
    else k_sum<double, false><<<g, 256, 0, s>>>((const double *)x, n, out1);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_sum_w_w2(const void *w, int dtype, int64_t n, double *out2, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "nbk_sum_w_w2: bad dtype %d", dtype);
    if (n <= 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    int g = nbk_grid_for(n, 256, 4);
    if (dtype == NBK_F4) k_sum<float, true><<<g, 256, 0, s>>>((const float *)w, n, out2);
    else k_sum<double, true><<<g, 256, 0, s>>>((const double *)w, n, out2);
    NBK_LAUNCHED();
    return NBK_OK;
}
