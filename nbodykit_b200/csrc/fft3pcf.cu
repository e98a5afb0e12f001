// FFT three-point correlation function of a periodic box (algorithms/fft3pcf.py: FFT3PCF; DESIGN.md 4.16):
//   nbk_fft3pcf_kernel_fill -- the real harmonic kernels K_lm,b(s) = Y_lm(u) 1_b(s) of one (l, radial bin b) for a run of
//                              m on the local x slab of a real mesh (the inputs of the kernel r2c transforms)
//   nbk_fft3pcf_gram        -- out[i][j] += sum_x w a_i b_j over two sets of resident real x-slab fields, register-blocked
//                              over the outer product (i <= j only when the two sets are the same)
//   nbk_fft3pcf_gram_tiles  -- the same over a list of 64-cell tiles, for weight fields that are zero outside them
//                              (algorithms/convfft3pcf.py: ConvolvedFFT3PCF; DESIGN.md 4.17)
//
// Built with --fmad=false: r = sqrt((sx^2 + sy^2) + sz^2) decides the bin of a grid separation, so no contraction may
// move a separation across an edge; the Y_lm polynomials and the Gram sums use explicit fma().
#include "common.cuh"

#include <math.h>

#define F3_MAX_L 10        // largest multipole (SimulationBox3PCF's max_ell)
#define F3_THREADS 256
#define F3_TILE 64         // cells per shared-memory tile of the Gram
#define F3_BLK 4           // each Gram thread owns a F3_BLK x F3_BLK block of (i, j)
#define F3_MAX_SET 32      // fields per set of the Gram (max_bins)

struct KernelParams {
    int64_t N[3];                                   // mesh sides
    int64_t x_start, x_n;                           // the local x slab
    double H[3];                                    // cell sides L_i / N_i
    double lo, hi;                                  // the bin: lo < r <= hi
    int ell, m0, nm;                                // fields m = m0 .. m0 + nm - 1 (signed real-harmonic index)
    int64_t nelem, ostride;                         // cells of the slab; elements between two output fields
    double coef[F3_MAX_L + 1][F3_MAX_L + 1];        // coef[|m|][k]: coefficient of uz^k in sqrt(4 pi) N_lm Q_lm
    double norm[2 * F3_MAX_L + 1];                  // per field of the run: 1 / sqrt(4 pi), times sqrt(2) for m != 0
};

// the separation index of grid index i on a side of n cells: i for 2 i <= n, else i - n, so that n_i lies in
// (-n/2, n/2] -- the half-open range of SimulationBox3PCF's periodic wrap
static __device__ __forceinline__ int64_t sep_index(int64_t i, int64_t n) { return (2 * i <= n) ? i : i - n; }

// One thread per cell of the slab (grid-stride).  s = (n_x H_x, n_y H_y, n_z H_z), r = sqrt((sx^2 + sy^2) + sz^2) in
// float64; a cell in the bin (lo < r <= hi, r > 0) gets, for every field of the run, the real orthonormal harmonic
//   m = 0: Y_l0,  m > 0: sqrt(2) Re y_lm,  m < 0: sqrt(2) Im y_l|m|,   y_lm = N_lm (ux + i uy)^m Q_lm(uz),  u = s / r
// evaluated in float64 and rounded once to the mesh precision; every other cell gets 0.
template <typename T>
__global__ void __launch_bounds__(F3_THREADS) k_fft3pcf_fill(KernelParams P, T *__restrict__ out) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < P.nelem; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t iz = e % P.N[2];
        const int64_t row = e / P.N[2];
        const int64_t iy = row % P.N[1], ix = P.x_start + row / P.N[1];
        const double sx = (double)sep_index(ix, P.N[0]) * P.H[0];
        const double sy = (double)sep_index(iy, P.N[1]) * P.H[1];
        const double sz = (double)sep_index(iz, P.N[2]) * P.H[2];
        const double r = sqrt((sx * sx + sy * sy) + sz * sz);
        const bool in = r > 0.0 && r > P.lo && r <= P.hi;
        T *o = out + e;
        if (!in) {
            for (int q = 0; q < P.nm; q++) o[q * P.ostride] = (T)0;
            continue;
        }
        const double ux = sx / r, uy = sy / r, uz = sz / r;
        // (ux + i uy)^|m| by repeated multiplication, restarted where |m| decreases along the run
        double er = 1.0, ei = 0.0;
        int mcur = 0;
        for (int q = 0; q < P.nm; q++) {
            const int m = P.m0 + q, am = m < 0 ? -m : m;
            if (am < mcur) {
                er = 1.0;
                ei = 0.0;
                mcur = 0;
            }
            while (mcur < am) {
                const double nr = er * ux - ei * uy;
                ei = er * uy + ei * ux;
                er = nr;
                mcur++;
            }
            // Q(uz) by Horner over the degree l - |m| polynomial
            const int deg = P.ell - am;
            double qv = P.coef[am][deg];
            for (int k = deg - 1; k >= 0; k--) qv = fma(qv, uz, P.coef[am][k]);
            const double v = (m >= 0 ? er : ei) * qv * P.norm[q];
            o[q * P.ostride] = (T)v;
        }
    }
}

// Block: the cell tiles blockIdx.x, blockIdx.x + gridDim.x, ...  A tile of F3_TILE cells of w and of every field of A
// and B (rows padded to multiples of F3_BLK with zeros) is staged in shared memory as float64, cell-major ([cell][row],
// odd row pitch: the lanes of a warp read neighbouring rows of one cell without bank conflicts).  Thread t owns the
// (i, j) block t % nblk and the cells t / nblk, t / nblk + ngroup, ... of each tile: per cell it forms w a_i once for
// its F3_BLK rows of A and adds (w a_i) b_j into F3_BLK^2 float64 registers.  SYM: B is A and only blocks with bi <= bj
// exist.  At the end the groups' partial blocks are summed in shared memory and each (i, j) gets one float64 atomic
// per block (diagonal blocks of SYM only add i <= j).  LIST: the block walks entries blockIdx.x, blockIdx.x + gridDim.x,
// ... of the tile list tiles[ntiles] instead of every tile (a tile left out must have w = 0 on all its cells).
template <typename T, bool SYM, bool LIST>
__global__ void __launch_bounds__(F3_THREADS) k_fft3pcf_gram(const T *__restrict__ w, const T *__restrict__ A,
                                                             int64_t astride, int na, const T *__restrict__ B,
                                                             int64_t bstride, int nb, int64_t ncell,
                                                             double *__restrict__ out, const int64_t *__restrict__ tiles,
                                                             int64_t ntiles) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double *s = reinterpret_cast<double *>(smem_raw);
    const int RA = (na + F3_BLK - 1) / F3_BLK * F3_BLK;
    const int RB = SYM ? 0 : (nb + F3_BLK - 1) / F3_BLK * F3_BLK;
    const int ld = RA + RB + 1;                      // odd pitch: row RA + RB holds w
    const int nbi = RA / F3_BLK, nbj = SYM ? nbi : RB / F3_BLK;
    const int nblk = SYM ? nbi * (nbi + 1) / 2 : nbi * nbj;
    const int ngroup = F3_THREADS / nblk;
    const int blk = threadIdx.x % nblk, grp = threadIdx.x / nblk;
    int bi, bj;
    if (SYM) {
        // blk -> (bi, bj), bi <= bj, row-major over the upper triangle
        bi = 0;
        int rest = blk;
        while (rest >= nbi - bi) {
            rest -= nbi - bi;
            bi++;
        }
        bj = bi + rest;
    } else {
        bi = blk / nbj;
        bj = blk - bi * nbj;
    }
    const int ra = bi * F3_BLK, rb = (SYM ? 0 : RA) + bj * F3_BLK;
    double acc[F3_BLK][F3_BLK];
#pragma unroll
    for (int i = 0; i < F3_BLK; i++)
#pragma unroll
        for (int j = 0; j < F3_BLK; j++) acc[i][j] = 0.0;
    const int nrow = RA + RB + 1;
    const int64_t nwalk = LIST ? ntiles : (ncell + F3_TILE - 1) / F3_TILE;
    for (int64_t it = blockIdx.x; it < nwalk; it += gridDim.x) {
        const int64_t c0 = (LIST ? tiles[it] : it) * F3_TILE;
        __syncthreads();
        for (int idx = threadIdx.x; idx < nrow * F3_TILE; idx += F3_THREADS) {
            const int r = idx / F3_TILE, cc = idx - r * F3_TILE;
            const int64_t c = c0 + cc;
            double v = 0.0;
            if (c < ncell) {
                if (r < RA) {
                    if (r < na) v = (double)A[r * astride + c];
                } else if (r < RA + RB) {
                    if (r - RA < nb) v = (double)B[(r - RA) * bstride + c];
                } else {
                    v = (double)w[c];
                }
            }
            s[cc * ld + r] = v;
        }
        __syncthreads();
        if (grp < ngroup) {
            for (int cc = grp; cc < F3_TILE; cc += ngroup) {
                const double *sc = s + cc * ld;
                const double wv = sc[ld - 1];
                double a[F3_BLK], b[F3_BLK];
#pragma unroll
                for (int i = 0; i < F3_BLK; i++) a[i] = wv * sc[ra + i];
#pragma unroll
                for (int j = 0; j < F3_BLK; j++) b[j] = sc[rb + j];
#pragma unroll
                for (int i = 0; i < F3_BLK; i++)
#pragma unroll
                    for (int j = 0; j < F3_BLK; j++) acc[i][j] = fma(a[i], b[j], acc[i][j]);
            }
        }
    }
    // the groups' partial blocks: [grp][blk][F3_BLK^2] (the launch sizes shared memory for this too)
    __syncthreads();
    const int BB = F3_BLK * F3_BLK;
    if (grp < ngroup) {
        double *p = s + ((size_t)grp * nblk + blk) * BB;
#pragma unroll
        for (int i = 0; i < F3_BLK; i++)
#pragma unroll
            for (int j = 0; j < F3_BLK; j++) p[i * F3_BLK + j] = acc[i][j];
    }
    __syncthreads();
    for (int e = threadIdx.x; e < nblk * BB; e += F3_THREADS) {
        const int b = e / BB, ij = e - b * BB;
        int pbi, pbj;
        if (SYM) {
            pbi = 0;
            int rest = b;
            while (rest >= nbi - pbi) {
                rest -= nbi - pbi;
                pbi++;
            }
            pbj = pbi + rest;
        } else {
            pbi = b / nbj;
            pbj = b - pbi * nbj;
        }
        const int i = pbi * F3_BLK + ij / F3_BLK, j = pbj * F3_BLK + ij % F3_BLK;
        if (i >= na || j >= nb || (SYM && i > j)) continue;
        double sum = 0.0;
        for (int g = 0; g < ngroup; g++) sum += s[((size_t)g * nblk + b) * BB + ij];
        atomicAdd(&out[(int64_t)i * nb + j], sum);
    }
}

extern "C" int nbk_fft3pcf_kernel_fill(void *out, int dtype, const int64_t *nmesh_host, const double *box_host,
                                       int64_t x_start, int64_t x_n, const double *edges_host, int nedges, int bin, int ell,
                                       int m0, int nm, const double *coef_host, int L, int64_t out_stride, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "fft3pcf_kernel_fill: bad dtype %d", dtype);
    NBK_CHECK_ARG(nmesh_host != nullptr && box_host != nullptr && edges_host != nullptr && coef_host != nullptr,
                  "fft3pcf_kernel_fill: null argument");
    NBK_CHECK_ARG(L >= 0 && L <= F3_MAX_L, "fft3pcf_kernel_fill: table of l <= %d (0 .. %d)", L, F3_MAX_L);
    NBK_CHECK_ARG(ell >= 0 && ell <= L, "fft3pcf_kernel_fill: l = %d outside the table (0 .. %d)", ell, L);
    NBK_CHECK_ARG(nm >= 0 && m0 >= -ell && m0 + nm <= ell + 1, "fft3pcf_kernel_fill: m = %d .. %d outside -%d .. %d", m0,
                  m0 + nm - 1, ell, ell);
    NBK_CHECK_ARG(nedges >= 2 && bin >= 0 && bin < nedges - 1, "fft3pcf_kernel_fill: bin %d of %d", bin, nedges - 1);
    KernelParams P;
    for (int d = 0; d < 3; d++) {
        NBK_CHECK_ARG(nmesh_host[d] > 0 && box_host[d] > 0, "fft3pcf_kernel_fill: bad mesh or box");
        P.N[d] = nmesh_host[d];
        P.H[d] = box_host[d] / (double)nmesh_host[d];
    }
    NBK_CHECK_ARG(x_start >= 0 && x_n >= 0 && x_start + x_n <= P.N[0], "fft3pcf_kernel_fill: bad x slab");
    NBK_CHECK_ARG(edges_host[bin + 1] > edges_host[bin], "fft3pcf_kernel_fill: the edges must increase");
    P.x_start = x_start;
    P.x_n = x_n;
    P.lo = edges_host[bin];
    P.hi = edges_host[bin + 1];
    P.ell = ell;
    P.m0 = m0;
    P.nm = nm;
    P.nelem = x_n * P.N[1] * P.N[2];
    NBK_CHECK_ARG(nm <= 1 || out_stride >= P.nelem, "fft3pcf_kernel_fill: output fields overlap");
    P.ostride = out_stride;
    // coefficient_table(L): row off(m) + l - m, off(m) = m (L + 1) - m (m - 1) / 2, L + 1 columns
    for (int m = 0; m <= F3_MAX_L; m++)
        for (int k = 0; k <= F3_MAX_L; k++) P.coef[m][k] = 0.0;
    for (int m = 0; m <= ell; m++) {
        const int row = m * (L + 1) - m * (m - 1) / 2 + ell - m;
        for (int k = 0; k <= ell - m; k++) {
            P.coef[m][k] = coef_host[(size_t)row * (L + 1) + k];
            NBK_CHECK_ARG(isfinite(P.coef[m][k]), "fft3pcf_kernel_fill: the coefficient table must be finite");
        }
    }
    const double inv_sqrt_4pi = 0.28209479177387814347403972578039;     // 1 / sqrt(4 pi)
    const double sqrt2 = 1.4142135623730950488016887242097;
    for (int q = 0; q < 2 * F3_MAX_L + 1; q++) P.norm[q] = 0.0;
    for (int q = 0; q < nm; q++) {
        const int m = m0 + q;
        P.norm[q] = m == 0 ? inv_sqrt_4pi : inv_sqrt_4pi * sqrt2;
    }
    if (P.nelem == 0 || nm == 0) return NBK_OK;
    NBK_CHECK_ARG(out != nullptr, "fft3pcf_kernel_fill: null output");
    cudaStream_t s = (cudaStream_t)stream;
    const int grid = nbk_grid_for(P.nelem, F3_THREADS, 8);
    if (dtype == NBK_F4) k_fft3pcf_fill<float><<<grid, F3_THREADS, 0, s>>>(P, (float *)out);
    else k_fft3pcf_fill<double><<<grid, F3_THREADS, 0, s>>>(P, (double *)out);
    NBK_LAUNCHED();
    return NBK_OK;
}

template <typename T, bool SYM, bool LIST>
static int launch_gram(const void *w, const void *A, int64_t astride, int na, const void *B, int64_t bstride, int nb,
                       int64_t ncell, const int64_t *tiles, int64_t ntiles, double *out, cudaStream_t s) {
    const int RA = (na + F3_BLK - 1) / F3_BLK * F3_BLK;
    const int RB = SYM ? 0 : (nb + F3_BLK - 1) / F3_BLK * F3_BLK;
    const int nbi = RA / F3_BLK, nbj = SYM ? nbi : RB / F3_BLK;
    const int nblk = SYM ? nbi * (nbi + 1) / 2 : nbi * nbj;
    const int ngroup = F3_THREADS / nblk;
    size_t smem = (size_t)F3_TILE * (RA + RB + 1) * sizeof(double);
    const size_t red = (size_t)ngroup * nblk * F3_BLK * F3_BLK * sizeof(double);
    if (red > smem) smem = red;
    NBK_CUDA(cudaFuncSetAttribute(k_fft3pcf_gram<T, SYM, LIST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 0;
    NBK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_fft3pcf_gram<T, SYM, LIST>, F3_THREADS, smem));
    if (occ < 1) occ = 1;
    const int64_t nwalk = LIST ? ntiles : (ncell + F3_TILE - 1) / F3_TILE;
    int64_t gx = (int64_t)NBK_SM_COUNT * occ;
    if (gx > nwalk) gx = nwalk;
    if (gx < 1) gx = 1;
    k_fft3pcf_gram<T, SYM, LIST><<<(unsigned)gx, F3_THREADS, smem, s>>>((const T *)w, (const T *)A, astride, na,
                                                                        (const T *)B, bstride, nb, ncell, out, tiles,
                                                                        ntiles);
    NBK_LAUNCHED();
    return NBK_OK;
}

template <bool LIST>
static int gram(const void *w, const void *A, int64_t a_stride, int na, const void *B, int64_t b_stride, int nb, int dtype,
                int64_t ncell, const int64_t *tiles, int64_t ntiles, double *out, void *stream) {
    const char *name = LIST ? "fft3pcf_gram_tiles" : "fft3pcf_gram";
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "%s: bad dtype %d", name, dtype);
    NBK_CHECK_ARG(na >= 1 && na <= F3_MAX_SET && nb >= 1 && nb <= F3_MAX_SET, "%s: %d x %d fields (1 .. %d each)", name,
                  na, nb, F3_MAX_SET);
    NBK_CHECK_ARG(ncell >= 0 && (na == 1 || a_stride >= ncell) && (nb == 1 || b_stride >= ncell),
                  "%s: bad field shape", name);
    NBK_CHECK_ARG(!LIST || (ntiles >= 0 && ntiles <= (ncell + F3_TILE - 1) / F3_TILE), "%s: %lld tiles of %lld",
                  name, (long long)ntiles, (long long)((ncell + F3_TILE - 1) / F3_TILE));
    if (ncell == 0 || (LIST && ntiles == 0)) return NBK_OK;
    NBK_CHECK_ARG(w != nullptr && A != nullptr && B != nullptr && out != nullptr && (!LIST || tiles != nullptr),
                  "%s: null pointer", name);
    cudaStream_t s = (cudaStream_t)stream;
    const bool sym = A == B && na == nb && (na == 1 || a_stride == b_stride);
    if (dtype == NBK_F4) {
        if (sym) return launch_gram<float, true, LIST>(w, A, a_stride, na, B, b_stride, nb, ncell, tiles, ntiles, out, s);
        return launch_gram<float, false, LIST>(w, A, a_stride, na, B, b_stride, nb, ncell, tiles, ntiles, out, s);
    }
    if (sym) return launch_gram<double, true, LIST>(w, A, a_stride, na, B, b_stride, nb, ncell, tiles, ntiles, out, s);
    return launch_gram<double, false, LIST>(w, A, a_stride, na, B, b_stride, nb, ncell, tiles, ntiles, out, s);
}

extern "C" int nbk_fft3pcf_gram(const void *w, const void *A, int64_t a_stride, int na, const void *B, int64_t b_stride,
                                int nb, int dtype, int64_t ncell, double *out, void *stream) {
    return gram<false>(w, A, a_stride, na, B, b_stride, nb, dtype, ncell, nullptr, 0, out, stream);
}

extern "C" int nbk_fft3pcf_gram_tiles(const void *w, const void *A, int64_t a_stride, int na, const void *B,
                                      int64_t b_stride, int nb, int dtype, int64_t ncell, const int64_t *tiles,
                                      int64_t ntiles, double *out, void *stream) {
    return gram<true>(w, A, a_stride, na, B, b_stride, nb, dtype, ncell, tiles, ntiles, out, stream);
}
