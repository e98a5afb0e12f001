// FFT bispectrum estimator (algorithms/bispectrum.py: FFTBispectrum; DESIGN.md 4.14):
//   nbk_bispec_fill       -- one read of the compressed Fourier slab writes c * 1_S or the f8 indicator 1_S for a
//                            range of k shells (the inputs of the shell c2r transforms)
//   nbk_bispec_fill_poles -- the same read writes c * L_ell(mu) * 1_S for a range of shells and several even ell (the
//                            inputs of the multipole fields W^ell; mu = k.los / |k| in nbk_power_bin's float32 arithmetic)
//   nbk_bispec_fill_cross -- one read of two compressed slabs writes scale * c * conj(d) * 1_S in float64 for a range of
//                            shells (the shot-noise fields H of ConvolvedFFTBispectrum)
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
#define BS_MAX_ELL 5     // ell = 0, 2, 4, 6, 8: the most multipoles one fill_poles call writes

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

// k_bispec_fill's shell rule, also returning the mode's float32 coordinates: the shell of element e of the slab relative
// to P.shell0 (-1: the k = 0 mode or outside every shell; values >= nshell are shells after the range).  k_bispec_fill
// keeps its own copy so that its generated code stays as it was.
__device__ __forceinline__ int fill_shell(const FillParams &P, int64_t e, float &kx, float &ky, float &kzv, float &k2) {
    const SlabGeom &g = P.g;
    const int kz = (int)(e % g.Nzc);
    const int64_t row = e / g.Nzc;
    const int i1 = (int)(row % g.D1), i0 = (int)(row / g.D1);
    int jx, jy, jz;
    slab_freqs(g, i0, i1, kz, jx, jy, jz);
    // (0 + kx^2) + ky^2, then + kz^2, in float32 as nbk_power_bin forms it
    kx = (float)jx * P.kf32[0];
    ky = (float)jy * P.kf32[1];
    kzv = (float)jz * P.kf32[2];
    const float kp2 = kx * kx + ky * ky;
    k2 = kp2 + kzv * kzv;
    const int b = nbk_k2_bin(P.k2e, P.nedge, (double)k2, (double)sqrtf(k2), P.kmin, P.inv_dk, P.uniform);
    int local = b - 1 - P.shell0;
    if (b < 1 || b >= P.nedge || (jx == 0 && jy == 0 && jz == 0)) local = -1;
    return local;
}

struct PoleParams {
    float los32[3];                     // the line of sight rounded to float32, as nbk_power_bin's coordinate mode 4
    int nell;
    int ells[BS_MAX_ELL];
};

// One thread per mode of the slab (grid-stride), the shell as in k_bispec_fill.  Output (q, s) -- multipole ells[q],
// shell shell0 + s -- starts (q nshell + s) ostride complex elements into `out` and holds c L_ell(mu) at the modes of
// its shell, 0 elsewhere.  mu = ((kx l0 + ky l1) + kz l2) / sqrtf(k2) in float32 (nbk_power_bin, coordinate mode 4),
// L_ell(mu) in float64, the product rounded once to the mesh precision.  L_ell is even for even ell, so the weighted
// half spectrum stays Hermitian.
template <typename T>
__global__ void __launch_bounds__(BS_THREADS)
k_bispec_fill_poles(const typename Cplx<T>::type *__restrict__ c, FillParams P, PoleParams L, void *__restrict__ out) {
    typedef typename Cplx<T>::type V2;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < P.nelem; e += (int64_t)gridDim.x * blockDim.x) {
        float kx, ky, kzv, k2;
        const int local = fill_shell(P, e, kx, ky, kzv, k2);
        const bool in = local >= 0 && local < P.nshell;
        double mu = 0.0, re = 0.0, im = 0.0;
        if (in) {
            const float lp = kx * L.los32[0] + ky * L.los32[1];
            mu = (double)((lp + kzv * L.los32[2]) / sqrtf(k2));
            const V2 v = c[e];
            re = (double)v.x;
            im = (double)v.y;
        }
        V2 *o = reinterpret_cast<V2 *>(out) + e;
        for (int q = 0; q < L.nell; q++) {
            V2 w;
            w.x = 0;
            w.y = 0;
            if (in) {
                const double f = legendre(L.ells[q], mu);
                w.x = (T)(re * f);
                w.y = (T)(im * f);
            }
            V2 *oq = o + (int64_t)q * P.nshell * P.ostride;
            for (int s = 0; s < P.nshell; s++) {
                V2 z;
                z.x = 0;
                z.y = 0;
                oq[s * P.ostride] = (s == local) ? w : z;
            }
        }
    }
}

// One thread per mode of the slab (grid-stride), k_bispec_fill's shell rule in its own copy (so that the generated
// code of k_bispec_fill and k_bispec_fill_poles stays as it was).  Output shell s starts s ostride complex float64
// elements into `out` and holds scale * c * conj(d) at the modes of its shell, 0 elsewhere: the product of the two
// mesh-precision values formed in float64.  For the spectra of two real fields the product is Hermitian.
template <typename T>
__global__ void __launch_bounds__(BS_THREADS)
k_bispec_fill_cross(const typename Cplx<T>::type *__restrict__ c, const typename Cplx<T>::type *__restrict__ d, FillParams P,
                    double scale, double2 *__restrict__ out) {
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
        double2 w = make_double2(0.0, 0.0);
        if (local >= 0 && local < P.nshell) {
            const V2 u = c[e], v = d[e];
            const double ur = (double)u.x, ui = (double)u.y, vr = (double)v.x, vi = (double)v.y;
            // (ur + i ui)(vr - i vi), every product rounded on its own (the file is built without FMA contraction)
            const double re = ur * vr + ui * vi;
            const double im = ui * vr - ur * vi;
            w = make_double2(re * scale, im * scale);
        }
        const double2 z = make_double2(0.0, 0.0);
        double2 *o = out + e;
        for (int s = 0; s < P.nshell; s++) o[s * P.ostride] = (s == local) ? w : z;
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

// the fill parameters of shells [shell0, shell0 + nshell) on this slab; nout output slabs out_stride apart
static int make_fill(int dtype, const int64_t *nmesh_host, const double *box_host, int layout, int64_t start, int64_t count,
                     const double *k2edges_host, int nedges, int shell0, int nshell, int nout, int64_t out_stride,
                     FillParams &P) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "bispec_fill: bad dtype %d", dtype);
    NBK_CHECK_ARG((layout & NBK_LAYOUT_FULLZ) == 0, "bispec_fill: the field must be Hermitian-compressed");
    NBK_CHECK_ARG(nedges >= 2 && nedges <= BS_MAX_SHELLS + 1, "bispec_fill: %d edges (2 .. %d)", nedges, BS_MAX_SHELLS + 1);
    NBK_CHECK_ARG(shell0 >= 0 && nshell >= 0 && shell0 + nshell <= nedges - 1, "bispec_fill: shells [%d,+%d) of %d", shell0,
                  nshell, nedges - 1);
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
    NBK_CHECK_ARG(nout <= 1 || out_stride >= P.nelem, "bispec_fill: output shells overlap");
    P.ostride = out_stride;
    return NBK_OK;
}

extern "C" int nbk_bispec_fill(const void *cplx, int dtype, const int64_t *nmesh_host, const double *box_host, int layout,
                               int64_t start, int64_t count, const double *k2edges_host, int nedges, int shell0, int nshell,
                               int indicator, void *out, int64_t out_stride, void *stream) {
    FillParams P;
    int rc = make_fill(dtype, nmesh_host, box_host, layout, start, count, k2edges_host, nedges, shell0, nshell, nshell,
                       out_stride, P);
    if (rc) return rc;
    NBK_CHECK_ARG(out != nullptr && (indicator || cplx != nullptr), "bispec_fill: null field");
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

extern "C" int nbk_bispec_fill_poles(const void *cplx, int dtype, const int64_t *nmesh_host, const double *box_host,
                                     int layout, int64_t start, int64_t count, const double *k2edges_host, int nedges,
                                     int shell0, int nshell, const double *los_host, const int *ells_host, int nell, void *out,
                                     int64_t out_stride, void *stream) {
    NBK_CHECK_ARG(nell >= 0 && nell <= BS_MAX_ELL, "bispec_fill_poles: %d multipoles (0 .. %d)", nell, BS_MAX_ELL);
    FillParams P;
    int rc = make_fill(dtype, nmesh_host, box_host, layout, start, count, k2edges_host, nedges, shell0, nshell,
                       nshell * nell, out_stride, P);
    if (rc) return rc;
    PoleParams L;
    L.nell = nell;
    for (int q = 0; q < nell; q++) {
        NBK_CHECK_ARG(ells_host[q] >= 0 && ells_host[q] <= 8 && ells_host[q] % 2 == 0,
                      "bispec_fill_poles: ell = %d (even, 0 .. 8: odd ell give an imaginary statistic)", ells_host[q]);
        L.ells[q] = ells_host[q];
    }
    for (int d = 0; d < 3; d++) L.los32[d] = (float)los_host[d];
    NBK_CHECK_ARG(out != nullptr && cplx != nullptr, "bispec_fill_poles: null field");
    if (P.nelem == 0 || nshell == 0 || nell == 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    const int grid = nbk_grid_for(P.nelem, BS_THREADS, 8);
    if (dtype == NBK_F4) {
        k_bispec_fill_poles<float><<<grid, BS_THREADS, 0, s>>>((const float2 *)cplx, P, L, out);
    } else {
        k_bispec_fill_poles<double><<<grid, BS_THREADS, 0, s>>>((const double2 *)cplx, P, L, out);
    }
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_bispec_fill_cross(const void *cplx, const void *cplx2, int dtype, const int64_t *nmesh_host,
                                     const double *box_host, int layout, int64_t start, int64_t count,
                                     const double *k2edges_host, int nedges, int shell0, int nshell, double scale, void *out,
                                     int64_t out_stride, void *stream) {
    FillParams P;
    int rc = make_fill(dtype, nmesh_host, box_host, layout, start, count, k2edges_host, nedges, shell0, nshell, nshell,
                       out_stride, P);
    if (rc) return rc;
    NBK_CHECK_ARG(out != nullptr && cplx != nullptr && cplx2 != nullptr, "bispec_fill_cross: null field");
    if (P.nelem == 0 || nshell == 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    const int grid = nbk_grid_for(P.nelem, BS_THREADS, 8);
    if (dtype == NBK_F4) {
        k_bispec_fill_cross<float><<<grid, BS_THREADS, 0, s>>>((const float2 *)cplx, (const float2 *)cplx2, P, scale,
                                                               (double2 *)out);
    } else {
        k_bispec_fill_cross<double><<<grid, BS_THREADS, 0, s>>>((const double2 *)cplx, (const double2 *)cplx2, P, scale,
                                                                (double2 *)out);
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
