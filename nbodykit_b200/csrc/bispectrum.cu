// FFT bispectrum estimator (algorithms/bispectrum.py: FFTBispectrum; DESIGN.md 4.14):
//   nbk_bispec_fill       -- one read of the compressed Fourier slab writes c * 1_S or the f8 indicator 1_S for a
//                            range of k shells (the inputs of the shell c2r transforms)
//   nbk_bispec_triple_sum -- sum_x f_i f_j f_l over resident real x-slab fields for a device list of slot triples
//
// Built with --fmad=false: the shell of a mode is decided by the float32 coordinate arithmetic of nbk_power_bin
// (kshell.cuh), so every FMA in this file is written out.
#include "common.cuh"
#include "kshell.cuh"

#define BS_MAX_SHELLS 64
#define BS_TILE 64       // cells per shared-memory tile of the triple sum
#define BS_TPT 4         // triples per thread of the triple sum
#define BS_THREADS 256

struct FillParams {
    SlabGeom g;
    float kf32[3];
    int nedge;                          // number of edges (shells + 1)
    double k2e[BS_MAX_SHELLS + 1];      // squared edges, as nbk_power_bin takes them
    double kmin, inv_dk;
    int uniform;
    int shell0, nshell;                 // shells [shell0, shell0 + nshell) are written
    int64_t nelem, ostride;             // elements of the slab, complex elements between two output shells
};

template <typename T> struct Cplx;
template <> struct Cplx<float> { typedef float2 type; };
template <> struct Cplx<double> { typedef double2 type; };

// One thread per mode of the slab (grid-stride).  The shell is the k bin nbk_power_bin gives the mode at float32
// coordinates, minus one (bin 0 lies below the first edge); the k = 0 mode belongs to no shell.  Every output shell
// of the range gets its value at this mode: the field value (or 1) in its own shell, 0 in the others.
template <typename T, bool IND>
__global__ void __launch_bounds__(BS_THREADS)
k_bispec_fill(const typename Cplx<T>::type *__restrict__ c, FillParams P, void *__restrict__ out) {
    typedef typename Cplx<T>::type V2;
    const SlabGeom &g = P.g;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < P.nelem; e += (int64_t)gridDim.x * blockDim.x) {
        const int kz = (int)(e % g.Nzc);
        const int64_t row = e / g.Nzc;
        const int i1 = (int)(row % g.D1), i0 = (int)(row / g.D1);
        int jx, jy, jz;
        slab_freqs(g, i0, i1, kz, jx, jy, jz);
        // (0 + kx^2) + ky^2, then + kz^2, in float32 as nbk_power_bin forms it
        const float kx = (float)jx * P.kf32[0], ky = (float)jy * P.kf32[1], kzv = (float)jz * P.kf32[2];
        const float kp2 = kx * kx + ky * ky;
        const float k2 = kp2 + kzv * kzv;
        const int b = nbk_k2_bin(P.k2e, P.nedge, (double)k2, (double)sqrtf(k2), P.kmin, P.inv_dk, P.uniform);
        int local = b - 1 - P.shell0;
        if (b < 1 || b >= P.nedge || (jx == 0 && jy == 0 && jz == 0)) local = -1;
        if (IND) {
            double2 *o = reinterpret_cast<double2 *>(out) + e;
            for (int s = 0; s < P.nshell; s++) o[s * P.ostride] = make_double2(s == local ? 1.0 : 0.0, 0.0);
        } else {
            const V2 v = c[e];
            V2 z;
            z.x = 0;
            z.y = 0;
            V2 *o = reinterpret_cast<V2 *>(out) + e;
            for (int s = 0; s < P.nshell; s++) o[s * P.ostride] = (s == local) ? v : z;
        }
    }
}

// Block (x, y): the cell tiles x, x + gridDim.x, ... and the triples [y BS_TPT BS_THREADS, (y + 1) BS_TPT BS_THREADS).
// A tile of BS_TILE cells of every resident field is staged in shared memory (rows padded by one element against bank
// conflicts); each thread then adds f_i f_j f_l over the tile for its BS_TPT triples, the product formed and the sum
// kept in float64.  One float64 atomic per triple and block at the end.
template <typename T>
__global__ void __launch_bounds__(BS_THREADS)
k_bispec_triple_sum(const T *__restrict__ f, int64_t fstride, int R, int64_t ncell, const int *__restrict__ tri,
                    int64_t ntri, double *__restrict__ out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    T *s = reinterpret_cast<T *>(smem_raw);
    const int ld = BS_TILE + 1;
    int ti[BS_TPT], tj[BS_TPT], tl[BS_TPT];
    double acc[BS_TPT];
#pragma unroll
    for (int k = 0; k < BS_TPT; k++) {
        const int64_t t = ((int64_t)blockIdx.y * BS_TPT + k) * BS_THREADS + threadIdx.x;
        const bool ok = t < ntri;
        ti[k] = ok ? tri[3 * t] * ld : -1;
        tj[k] = ok ? tri[3 * t + 1] * ld : 0;
        tl[k] = ok ? tri[3 * t + 2] * ld : 0;
        acc[k] = 0.0;
    }
    const int64_t ntile = (ncell + BS_TILE - 1) / BS_TILE;
    for (int64_t tile = blockIdx.x; tile < ntile; tile += gridDim.x) {
        const int64_t c0 = tile * BS_TILE;
        __syncthreads();
        for (int idx = threadIdx.x; idx < R * BS_TILE; idx += BS_THREADS) {
            const int r = idx / BS_TILE, cc = idx - r * BS_TILE;
            s[r * ld + cc] = (c0 + cc < ncell) ? f[r * fstride + c0 + cc] : (T)0;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BS_TPT; k++) {
            if (ti[k] < 0) continue;
            const T *a = s + ti[k], *b = s + tj[k], *d = s + tl[k];
            double sum = 0.0;
#pragma unroll 8
            for (int cc = 0; cc < BS_TILE; cc++) sum = fma((double)a[cc] * (double)b[cc], (double)d[cc], sum);
            acc[k] += sum;
        }
    }
#pragma unroll
    for (int k = 0; k < BS_TPT; k++)
        if (ti[k] >= 0) atomicAdd(&out[((int64_t)blockIdx.y * BS_TPT + k) * BS_THREADS + threadIdx.x], acc[k]);
}

extern "C" int nbk_bispec_max_shells(void) { return BS_MAX_SHELLS; }

extern "C" int nbk_bispec_fill(const void *cplx, int dtype, const int64_t *nmesh_host, const double *box_host, int layout,
                               int64_t start, int64_t count, const double *k2edges_host, int nedges, int shell0, int nshell,
                               int indicator, void *out, int64_t out_stride, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "bispec_fill: bad dtype %d", dtype);
    NBK_CHECK_ARG((layout & NBK_LAYOUT_FULLZ) == 0, "bispec_fill: the field must be Hermitian-compressed");
    NBK_CHECK_ARG(nedges >= 2 && nedges <= BS_MAX_SHELLS + 1, "bispec_fill: %d edges (2 .. %d)", nedges, BS_MAX_SHELLS + 1);
    NBK_CHECK_ARG(shell0 >= 0 && nshell >= 0 && shell0 + nshell <= nedges - 1, "bispec_fill: shells [%d,+%d) of %d", shell0,
                  nshell, nedges - 1);
    NBK_CHECK_ARG(out != nullptr && (indicator || cplx != nullptr), "bispec_fill: null field");
    FillParams P;
    int rc = make_slab(nmesh_host, layout, start, count, 1, P.g);
    if (rc) return rc;
    const double TWO_PI = 6.283185307179586476925286766559;
    for (int d = 0; d < 3; d++) {
        NBK_CHECK_ARG(box_host[d] > 0, "bispec_fill: bad BoxSize");
        P.kf32[d] = (float)(TWO_PI / box_host[d]);
    }
    for (int i = 0; i < nedges; i++) {
        P.k2e[i] = k2edges_host[i];
        NBK_CHECK_ARG(i == 0 || P.k2e[i] > P.k2e[i - 1], "bispec_fill: the squared edges must increase");
    }
    P.nedge = nedges;
    P.uniform = nbk_k2_uniform(P.k2e, nedges - 1, &P.kmin, &P.inv_dk);
    P.shell0 = shell0;
    P.nshell = nshell;
    P.nelem = (int64_t)P.g.count * P.g.D1 * P.g.Nzc;
    NBK_CHECK_ARG(nshell <= 1 || out_stride >= P.nelem, "bispec_fill: output shells overlap");
    P.ostride = out_stride;
    if (P.nelem == 0 || nshell == 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    const int grid = nbk_grid_for(P.nelem, BS_THREADS, 8);
    if (indicator) {
        k_bispec_fill<double, true><<<grid, BS_THREADS, 0, s>>>(nullptr, P, out);
    } else if (dtype == NBK_F4) {
        k_bispec_fill<float, false><<<grid, BS_THREADS, 0, s>>>((const float2 *)cplx, P, out);
    } else {
        k_bispec_fill<double, false><<<grid, BS_THREADS, 0, s>>>((const double2 *)cplx, P, out);
    }
    NBK_LAUNCHED();
    return NBK_OK;
}

template <typename T>
static int launch_triple_sum(const void *fields, int64_t fstride, int R, int64_t ncell, const int *tri, int64_t ntri,
                             double *out, cudaStream_t s) {
    const size_t smem = (size_t)R * (BS_TILE + 1) * sizeof(T);
    NBK_CUDA(cudaFuncSetAttribute(k_bispec_triple_sum<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t per = (int64_t)BS_TPT * BS_THREADS;
    const int64_t gy = (ntri + per - 1) / per;
    NBK_CHECK_ARG(gy <= 65535, "bispec_triple_sum: too many triples (%lld)", (long long)ntri);
    int occ = 0;
    NBK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_bispec_triple_sum<T>, BS_THREADS, smem));
    if (occ < 1) occ = 1;
    const int64_t ntile = (ncell + BS_TILE - 1) / BS_TILE;
    int64_t gx = ((int64_t)NBK_SM_COUNT * occ + gy - 1) / gy;
    if (gx > ntile) gx = ntile;
    if (gx < 1) gx = 1;
    k_bispec_triple_sum<T><<<dim3((unsigned)gx, (unsigned)gy), BS_THREADS, smem, s>>>((const T *)fields, fstride, R, ncell, tri,
                                                                                      ntri, out);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_bispec_triple_sum(const void *fields, int dtype, int64_t field_stride, int nfield, int64_t ncell,
                                     const int *triples, int64_t ntri, double *out, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "bispec_triple_sum: bad dtype %d", dtype);
    NBK_CHECK_ARG(nfield >= 1 && nfield <= BS_MAX_SHELLS, "bispec_triple_sum: %d resident fields (1 .. %d)", nfield,
                  BS_MAX_SHELLS);
    NBK_CHECK_ARG(ncell >= 0 && ntri >= 0 && (nfield == 1 || field_stride >= ncell), "bispec_triple_sum: bad field shape");
    if (ncell == 0 || ntri == 0) return NBK_OK;
    NBK_CHECK_ARG(fields != nullptr && triples != nullptr && out != nullptr, "bispec_triple_sum: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == NBK_F4) return launch_triple_sum<float>(fields, field_stride, nfield, ncell, triples, ntri, out, s);
    return launch_triple_sum<double>(fields, field_stride, nfield, ncell, triples, ntri, out, s);
}
