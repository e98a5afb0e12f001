// cuFFT-free 3-D real<->complex FFT (RealField.r2c / ComplexField.c2r: base/mesh.py:228,237;
// source/mesh/catalog.py:341-351).  Forward is normalised by 1/prod(N), backward is not
// (source/mesh/array.py:36-37, fftpower.py:126-128).
// c2r contract: for ANY half spectrum X [Nx][Ny][Nz/2+1] (no symmetry assumed) the result is irfftn(X, s=N) * prod(N),
// the rule of numpy / scipy irfftn and of FFTW's c2r: complex inverses along x and y, then a real inverse along z that
// drops the imaginary parts of the kz = 0 entry and, for even Nz, of the kz = Nz/2 entry.  Every inverse z pass (power
// of two, mixed radix, Bluestein; even and odd Nz) makes those entries real before it uses them.
//
// Structure: three line passes, each one read + one write of the field (HBM-bound):
//   z pass  : rows are contiguous; real row of Nz -> packed complex FFT of Nz/2 -> Nz/2+1 modes
//   y pass  : lines strided by Nzc, tiles of B adjacent kz columns  (B * sizeof(cplx) = 128-byte runs)
//   x pass  : lines strided by Ny*Nzc, tiles of B adjacent (y,kz) elements
// Default kernels (round 2), built around the copy engine so that the warps only run butterflies:
//   k_fft_lines_tma   lines of 256 / 512 / 1024: row groups stream through a ring of shared-memory slots as 4-D tensor-map
//                     boxes (cp.async.bulk.tensor + mbarrier), one 64-point FFT per warp, one radix-R combine per tile
//   k_fft_z_r2c_tma   rows of 256 / 512 / 1024 reals: warp-per-row, private ring of row buffers filled by 1-D bulk copies
//   k_fft_zy_r2c_pipe the forward z and y passes of c16 fields where both of the above apply, pipelined plane by plane
//                     so that the y tiles read the z rows from L2 (same device functions, same bits)
// Older families, still serving the other lengths, c8 lines whose rows are not 16-byte aligned and the backward z pass:
// the register-I/O kernels for lines of 64 and more (k_fft_lines_rg, k_fft_z_r2c_rg: first radix-8 stage straight from
// global memory, last stage straight to the digit-reversed frequency rows, [N][B+1] padded tiles in between) and the
// shared-memory kernels (k_fft_lines with cp.async double buffering for lines below 64, k_fft_z_r2c, k_fft_z_c2r).
// Decimation-in-frequency radix-8 butterflies in registers throughout (+ one radix-4 / radix-2 stage for the remainder of
// log2 N).  Twiddles: f8-accurate table built on the device with sincospi, staged in shared memory.  Sizes: 2^k.
// Sides that are products of 2, 3, 5 and 7 (Nx, Ny <= 4096; Nz <= 8192 even, <= 4095 odd) go through the separate
// mixed-radix entry points at the end of this file (k_fft_lines_mixed, k_fft_z_mixed; nbk_r2c_mixed / nbk_c2r_mixed), and
// axes whose side has a larger prime factor through the Bluestein passes after them (k_fft_lines_bluestein,
// k_fft_z_bluestein), which reuse the mixed-radix stages for their convolution.
#include "common.cuh"
#include "kshell.cuh"
#include <cuda.h>      // CUtensorMap types only: the encoder comes from cudaGetDriverEntryPoint (no -lcuda)
#include <map>
#include <mutex>
#include <tuple>
#include <stdlib.h>
#include <string.h>

template <typename T> struct C2;
template <> struct C2<float> { typedef float2 type; };
template <> struct C2<double> { typedef double2 type; };

template <typename C> __device__ __forceinline__ C cadd(C a, C b) { return C{a.x + b.x, a.y + b.y}; }
template <typename C> __device__ __forceinline__ C csub(C a, C b) { return C{a.x - b.x, a.y - b.y}; }
template <typename C> __device__ __forceinline__ C cmul(C a, C b) {
    return C{a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x};
}
template <typename C> __device__ __forceinline__ C cconj(C a) { return C{a.x, -a.y}; }
template <typename C> __device__ __forceinline__ C cmuli_neg(C a) { return C{a.y, -a.x}; }  // a * (-i)

// Stage plan: radix-8 stages, then one radix-4 or radix-2 stage for the remainder of log2(N).
// position (in the in-place DIF output) of frequency k = mixed-radix digit reversal
__device__ __forceinline__ int pos_of_freq(int k, int N, int log2n) {
    int rem = k, base = N, pos = 0;
    const int n8 = log2n / 3, r = log2n - 3 * n8;
    for (int s = 0; s < n8; s++) {
        int d = rem & 7;
        rem >>= 3;
        base >>= 3;
        pos += d * base;
    }
    if (r == 2) pos += (rem & 3);        // base == 4 -> base/4 == 1
    else if (r == 1) pos += (rem & 1);
    return pos;
}

template <typename C> struct Sqrt1_2;
template <> struct Sqrt1_2<float2> { static __device__ __forceinline__ float v() { return 0.70710678118654752440f; } };
template <> struct Sqrt1_2<double2> { static __device__ __forceinline__ double v() { return 0.70710678118654752440; } };

// 4-point DFT (forward): X0 = c0+c1, X1 = c2+c3, X2 = c0-c1, X3 = c2-c3
template <typename C>
__device__ __forceinline__ void dft4(C &a0, C &a1, C &a2, C &a3) {
    C c0 = cadd(a0, a2), c1 = cadd(a1, a3), c2 = csub(a0, a2), c3 = cmuli_neg(csub(a1, a3));
    a0 = cadd(c0, c1);
    a1 = cadd(c2, c3);
    a2 = csub(c0, c1);
    a3 = csub(c2, c3);
}

// Shared-memory address (in elements) of line element e, column b.  Rows are padded to B+1 elements; with SKEW an
// extra element is inserted every N/8 rows, so that the digit-reversed rows 0, N/8, 2N/8, ... which consecutive
// output frequencies live in fall into different banks (the z passes read the tile with lanes along frequency).
template <int B, bool SKEW>
__device__ __forceinline__ int saddr(int e, int sk) { return e * (B + 1) + (SKEW ? (e >> sk) : 0); }

// In-place forward DIF FFT of B side-by-side lines of length N held at sm[saddr(n) + b].
// tw[k] = exp(-2 pi i k / N), k < N (shared or global memory).  All threads of the CTA must call.
// Each radix-8 butterfly lives in registers: 8 LDS + 8 STS per 8 points per stage (3 stages at N = 512).
template <typename C, int B, bool SKEW = false>
__device__ __forceinline__ void fft_tile(C *sm, const C *__restrict__ tw, int N, int log2n) {
    const int T = blockDim.x;
    const int sk = log2n >= 3 ? log2n - 3 : 31;
    const int n8 = log2n / 3, rrem = log2n - 3 * n8;
    int Ns = N;
    int lq = log2n;
    for (int s = 0; s < n8; s++) {
        const int Q = Ns >> 3;
        lq -= 3;                       // log2(Q)
        const int tws = N / Ns;
        const int work = (N >> 3) * B;
        for (int w = threadIdx.x; w < work; w += T) {
            int b = w % B;
            int t = w / B;
            int blk = t >> lq, q = t & (Q - 1);
            const int e0 = blk * Ns + q;
            C *p0 = sm + saddr<B, SKEW>(e0, sk) + b, *p1 = sm + saddr<B, SKEW>(e0 + Q, sk) + b;
            C *p2 = sm + saddr<B, SKEW>(e0 + 2 * Q, sk) + b, *p3 = sm + saddr<B, SKEW>(e0 + 3 * Q, sk) + b;
            C *p4 = sm + saddr<B, SKEW>(e0 + 4 * Q, sk) + b, *p5 = sm + saddr<B, SKEW>(e0 + 5 * Q, sk) + b;
            C *p6 = sm + saddr<B, SKEW>(e0 + 6 * Q, sk) + b, *p7 = sm + saddr<B, SKEW>(e0 + 7 * Q, sk) + b;
            C a0 = *p0, a1 = *p1, a2 = *p2, a3 = *p3, a4 = *p4, a5 = *p5, a6 = *p6, a7 = *p7;
            // level 1: b_m = a_m + a_{m+4}; b_{m+4} = (a_m - a_{m+4}) W8^m
            C b0 = cadd(a0, a4), b1 = cadd(a1, a5), b2 = cadd(a2, a6), b3 = cadd(a3, a7);
            C b4 = csub(a0, a4), d5 = csub(a1, a5), d6 = csub(a2, a6), d7 = csub(a3, a7);
            const auto h = Sqrt1_2<C>::v();
            C b5 = C{(d5.x + d5.y) * h, (d5.y - d5.x) * h};     // * (1 - i)/sqrt2
            C b6 = cmuli_neg(d6);                                // * (-i)
            C b7 = C{(d7.y - d7.x) * h, -(d7.x + d7.y) * h};    // * (-1 - i)/sqrt2
            dft4(b0, b1, b2, b3);      // -> y0, y2, y4, y6
            dft4(b4, b5, b6, b7);      // -> y1, y3, y5, y7
            if (Q > 1) {
                int ti = q * tws;
                b4 = cmul(b4, tw[ti]);
                b1 = cmul(b1, tw[2 * ti]);
                b5 = cmul(b5, tw[3 * ti]);
                b2 = cmul(b2, tw[4 * ti]);
                b6 = cmul(b6, tw[5 * ti]);
                b3 = cmul(b3, tw[6 * ti]);
                b7 = cmul(b7, tw[7 * ti]);
            }
            *p0 = b0; *p1 = b4; *p2 = b1; *p3 = b5; *p4 = b2; *p5 = b6; *p6 = b3; *p7 = b7;
        }
        __syncthreads();
        Ns = Q;
    }
    if (rrem == 2) {   // Ns == 4, Q == 1: no twiddles
        const int work = (N >> 2) * B;
        for (int w = threadIdx.x; w < work; w += T) {
            int b = w % B;
            int t = w / B;
            C *p0 = sm + saddr<B, SKEW>(4 * t, sk) + b, *p1 = sm + saddr<B, SKEW>(4 * t + 1, sk) + b;
            C *p2 = sm + saddr<B, SKEW>(4 * t + 2, sk) + b, *p3 = sm + saddr<B, SKEW>(4 * t + 3, sk) + b;
            C a0 = *p0, a1 = *p1, a2 = *p2, a3 = *p3;
            dft4(a0, a1, a2, a3);
            *p0 = a0; *p1 = a1; *p2 = a2; *p3 = a3;
        }
        __syncthreads();
    } else if (rrem == 1) {  // Ns == 2
        const int work = (N >> 1) * B;
        for (int w = threadIdx.x; w < work; w += T) {
            int b = w % B;
            int t = w / B;
            C *p0 = sm + saddr<B, SKEW>(2 * t, sk) + b, *p1 = sm + saddr<B, SKEW>(2 * t + 1, sk) + b;
            C a0 = *p0, a1 = *p1;
            *p0 = cadd(a0, a1);
            *p1 = csub(a0, a1);
        }
        __syncthreads();
    }
}

// copy the twiddle table into shared memory (after the tile); returns the shared pointer
template <typename C>
__device__ __forceinline__ const C *stage_twiddles(C *dst, const C *__restrict__ tw, int N) {
    for (int i = threadIdx.x; i < N; i += blockDim.x) dst[i] = tw[i];
    __syncthreads();
    return dst;
}

// ---------------------------------------------------------------------------------------------
// strided line pass (y and x passes), in place.  element(outer, n, inner) =
//   data[outer*outer_stride + n*line_stride + inner],  inner < n_inner contiguous.
// ---------------------------------------------------------------------------------------------
// 16- / 8-byte asynchronous global -> shared copies (LDGSTS): the next tile streams in while this one is transformed
__device__ __forceinline__ void cp_async_elem(double2 *sdst, const double2 *gsrc) {
    unsigned sa = (unsigned)__cvta_generic_to_shared(sdst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(sa), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_elem(float2 *sdst, const float2 *gsrc) {
    unsigned sa = (unsigned)__cvta_generic_to_shared(sdst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" :: "r"(sa), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N_> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N_) : "memory"); }

// strided tile -> shared [N][B+1]; columns beyond the valid width are zero-filled with plain stores
template <typename C, int B>
__device__ __forceinline__ void prefetch_tile(C *sm, const C *base, int N, int64_t line_stride, int bvalid) {
    constexpr int pitch = B + 1;
    for (int w = threadIdx.x; w < N * B; w += blockDim.x) {
        int b = w % B, n = w / B;
        if (b < bvalid) cp_async_elem(&sm[n * pitch + b], base + (int64_t)n * line_stride + b);
        else sm[n * pitch + b] = C{0, 0};
    }
}

template <typename T, int B>
__global__ void __launch_bounds__(512)
k_fft_lines(const typename C2<T>::type *src, typename C2<T>::type *dst, const typename C2<T>::type *__restrict__ tw,
            int N, int log2n, int64_t line_stride, int64_t n_inner, int64_t tiles_inner, int64_t n_tiles, int64_t outer_stride,
            int inverse, T scale) {
    typedef typename C2<T>::type C;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    // shared: buf[2][N][B+1] | twiddles[N]  -- two tile buffers: tile i+1 is prefetched with cp.async while tile i is
    // transformed and written back
    C *buf0 = reinterpret_cast<C *>(smem_raw);
    constexpr int pitch = B + 1;
    C *buf1 = buf0 + (size_t)N * pitch;
    const int T_ = blockDim.x;
    tw = stage_twiddles<C>(buf1 + (size_t)N * pitch, tw, N);
    int64_t tile = blockIdx.x;
    if (tile < n_tiles) {
        int64_t outer = tile / tiles_inner;
        int64_t inner0 = (tile - outer * tiles_inner) * B;
        int bvalid = (int)((n_inner - inner0) < B ? (n_inner - inner0) : B);
        prefetch_tile<C, B>(buf0, src + outer * outer_stride + inner0, N, line_stride, bvalid);
    }
    cp_async_commit();
    int cur = 0;
    for (; tile < n_tiles; tile += gridDim.x, cur ^= 1) {
        C *sm = cur ? buf1 : buf0;
        int64_t outer = tile / tiles_inner;
        int64_t inner0 = (tile - outer * tiles_inner) * B;
        C *obase = dst + outer * outer_stride + inner0;      // dst == src: in place (a CTA owns its tile)
        int bvalid = (int)((n_inner - inner0) < B ? (n_inner - inner0) : B);
        int64_t nxt = tile + gridDim.x;
        if (nxt < n_tiles) {
            int64_t o2 = nxt / tiles_inner;
            int64_t i2 = (nxt - o2 * tiles_inner) * B;
            int bv2 = (int)((n_inner - i2) < B ? (n_inner - i2) : B);
            prefetch_tile<C, B>(cur ? buf0 : buf1, src + o2 * outer_stride + i2, N, line_stride, bv2);
        }
        cp_async_commit();
        cp_async_wait<1>();          // this tile's copies have landed (the prefetch may still be in flight)
        __syncthreads();
        if (inverse) {
            for (int w = threadIdx.x; w < N * B; w += T_) { int b = w % B, n = w / B; sm[n * pitch + b].y = -sm[n * pitch + b].y; }
            __syncthreads();
        }
        fft_tile<C, B>(sm, tw, N, log2n);
        for (int w = threadIdx.x; w < N * B; w += T_) {
            int b = w % B, k = w / B;
            if (b < bvalid) {
                C v = sm[pos_of_freq(k, N, log2n) * pitch + b];
                if (inverse) v.y = -v.y;
                v.x *= scale;
                v.y *= scale;
                obase[(int64_t)k * line_stride + b] = v;
            }
        }
        __syncthreads();             // everyone is done with `sm` before the next prefetch overwrites it
    }
    cp_async_wait<0>();
}
// ---------------------------------------------------------------------------------------------
// Fused line pass + slab transpose over peer memory (P > 1).  Lines of length N run along the SECOND stored axis
// of the local slab src[n_outer][N][n_inner] (the y pass of r2c on [x_n][Ny][Nzc], or the inverse x pass of c2r on
// [y_n][Nx][Nzc]).  Output frequency k belongs to rank p = k / (N/P); instead of writing the slab back, packing,
// all-to-all and unpacking, the store phase writes each 64..128-byte kz run straight into rank p's transposed
// field through its NVLink-mapped pointer:
//     peer[p][ ((k % (N/P)) * (n_outer*P) + outer_start + outer) * n_inner + kz ]
// (peer[rank] is the local buffer).  The caller brackets the launch with cross-rank barriers.
// ---------------------------------------------------------------------------------------------
#define NBK_MAX_PEERS 16
template <typename C> struct PeerPtrs { C *p[NBK_MAX_PEERS]; };

template <typename T, int B>
__global__ void __launch_bounds__(256)
k_fft_lines_scatter(const typename C2<T>::type *__restrict__ src, PeerPtrs<typename C2<T>::type> peers,
                    const typename C2<T>::type *__restrict__ tw, int N, int log2n, int64_t n_inner, int64_t tiles_inner,
                    int64_t n_tiles, int n_per, int64_t d_total, int64_t outer_start, int inverse, T scale) {
    typedef typename C2<T>::type C;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    C *sm = reinterpret_cast<C *>(smem_raw);
    constexpr int pitch = B + 1;
    const int T_ = blockDim.x;
    tw = stage_twiddles<C>(sm + N * pitch, tw, N);
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        int64_t outer = tile / tiles_inner;
        int64_t inner0 = (tile - outer * tiles_inner) * B;
        const C *base = src + outer * (int64_t)N * n_inner + inner0;
        int bvalid = (int)((n_inner - inner0) < B ? (n_inner - inner0) : B);
        for (int w = threadIdx.x; w < N * B; w += T_) {
            int b = w % B, n = w / B;
            C v = C{0, 0};
            if (b < bvalid) v = base[(int64_t)n * n_inner + b];
            if (inverse) v.y = -v.y;
            sm[n * pitch + b] = v;
        }
        __syncthreads();
        fft_tile<C, B>(sm, tw, N, log2n);
        for (int w = threadIdx.x; w < N * B; w += T_) {
            int b = w % B, k = w / B;
            if (b < bvalid) {
                C v = sm[pos_of_freq(k, N, log2n) * pitch + b];
                if (inverse) v.y = -v.y;
                v.x *= scale;
                v.y *= scale;
                int p = k / n_per, kl = k - p * n_per;
                peers.p[p][((int64_t)kl * d_total + outer_start + outer) * n_inner + inner0 + b] = v;
            }
        }
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------
// Register-I/O line pass (N >= 64).  The first radix-8 stage loads its 8 inputs per butterfly straight from global
// memory (rows q + k*N/8, B adjacent columns per row = one 128-byte run per quarter warp), and the last stage
// writes its outputs straight to their digit-reversed frequency rows; shared memory only carries the exchanges
// between stages (4 instead of 8 shared accesses per element at N = 512, and no copy loops).  One tile buffer per
// CTA, so 2-3 CTAs share an SM and one CTA's global phase overlaps another's butterflies.
// PEER: the store goes to the NVLink-mapped transposed field of rank k / n_per (see k_fft_lines_scatter).
// ---------------------------------------------------------------------------------------------
template <typename C>
__device__ __forceinline__ void radix8(C (&a)[8]) {   // in: a[j] = x_j ; out: a[m] = X_m (8-point forward DFT)
    C b0 = cadd(a[0], a[4]), b1 = cadd(a[1], a[5]), b2 = cadd(a[2], a[6]), b3 = cadd(a[3], a[7]);
    C b4 = csub(a[0], a[4]), d5 = csub(a[1], a[5]), d6 = csub(a[2], a[6]), d7 = csub(a[3], a[7]);
    const auto h = Sqrt1_2<C>::v();
    C b5 = C{(d5.x + d5.y) * h, (d5.y - d5.x) * h};
    C b6 = cmuli_neg(d6);
    C b7 = C{(d7.y - d7.x) * h, -(d7.x + d7.y) * h};
    dft4(b0, b1, b2, b3);      // -> X0, X2, X4, X6
    dft4(b4, b5, b6, b7);      // -> X1, X3, X5, X7
    a[0] = b0; a[1] = b4; a[2] = b1; a[3] = b5; a[4] = b2; a[5] = b6; a[6] = b3; a[7] = b7;
}

__device__ __forceinline__ int rev8(int t, int ndig) {   // reverse the ndig base-8 digits of t
    int r = 0;
    for (int i = 0; i < ndig; i++) { r = (r << 3) | (t & 7); t >>= 3; }
    return r;
}

template <typename T, int B, bool PEER, int NT>
__global__ void __launch_bounds__(NT, 512 / NT)
k_fft_lines_rg(const typename C2<T>::type *src, typename C2<T>::type *dst, PeerPtrs<typename C2<T>::type> peers,
               const typename C2<T>::type *__restrict__ tw, int N, int log2n, int64_t line_stride, int64_t n_inner,
               int64_t tiles_inner, int64_t n_tiles, int64_t outer_stride, int n_per, int64_t d_total,
               int64_t outer_start, int inverse, T scale) {
    typedef typename C2<T>::type C;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    C *sm = reinterpret_cast<C *>(smem_raw);
    constexpr int pitch = B + 1;
    const int T_ = blockDim.x;
    tw = stage_twiddles<C>(sm + (size_t)N * pitch, tw, N);
    const int n8 = log2n / 3, rrem = log2n - 3 * n8;
    const int Q1 = N >> 3;
    const T sgn = inverse ? (T)-1 : (T)1;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        int64_t outer = tile / tiles_inner;
        int64_t inner0 = (tile - outer * tiles_inner) * B;
        const C *ibase = src + outer * outer_stride + inner0;
        int bvalid = (int)((n_inner - inner0) < B ? (n_inner - inner0) : B);
        // ---- first stage: global -> registers -> shared
        for (int w = threadIdx.x; w < Q1 * B; w += T_) {
            int b = w % B, q = w / B;
            C a[8];
            if (b < bvalid) {
                const C *g = ibase + (int64_t)q * line_stride + b;
#pragma unroll
                for (int j = 0; j < 8; j++) a[j] = g[(int64_t)j * Q1 * line_stride];
            } else {
#pragma unroll
                for (int j = 0; j < 8; j++) a[j] = C{0, 0};
            }
#pragma unroll
            for (int j = 0; j < 8; j++) a[j].y *= sgn;
            radix8(a);
            C *o = sm + q * pitch + b;
            o[0] = a[0];
#pragma unroll
            for (int m = 1; m < 8; m++) o[m * Q1 * pitch] = cmul(a[m], tw[m * q]);
        }
        __syncthreads();
        // ---- middle stages, in place in shared memory
        {
            const int last8 = rrem ? n8 : n8 - 1;    // radix-8 stages [1, last8) are exchanged through shared memory
            int Ns = Q1, lq = log2n - 3;
            for (int s = 1; s < last8; s++) {
                const int Q = Ns >> 3;
                lq -= 3;
                const int tws = N / Ns;
                for (int w = threadIdx.x; w < Q1 * B; w += T_) {
                    int b = w % B, t = w / B;
                    int blk = t >> lq, q = t & (Q - 1);
                    C *p = sm + (blk * Ns + q) * pitch + b;
                    C a[8];
#pragma unroll
                    for (int j = 0; j < 8; j++) a[j] = p[j * Q * pitch];
                    radix8(a);
                    int ti = q * tws;
                    p[0] = a[0];
#pragma unroll
                    for (int m = 1; m < 8; m++) p[m * Q * pitch] = cmul(a[m], tw[m * ti]);
                }
                __syncthreads();
                Ns = Q;
            }
        }
        // ---- last stage: shared -> registers -> global (frequency rows)
        const int R = rrem == 0 ? 8 : (rrem == 2 ? 4 : 2);
        const int NR = N / R;                 // butterflies per line, and the frequency step between its outputs
        const int ndig = rrem == 0 ? n8 - 1 : n8;
        for (int w = threadIdx.x; w < NR * B; w += T_) {
            int b = w % B, t = w / B;
            const C *p = sm + (t * R) * pitch + b;
            C a[8];
            if (R == 8) {
#pragma unroll
                for (int j = 0; j < 8; j++) a[j] = p[j * pitch];
                radix8(a);
            } else if (R == 4) {
                a[0] = p[0]; a[1] = p[pitch]; a[2] = p[2 * pitch]; a[3] = p[3 * pitch];
                dft4(a[0], a[1], a[2], a[3]);
            } else {
                C x0 = p[0], x1 = p[pitch];
                a[0] = cadd(x0, x1);
                a[1] = csub(x0, x1);
            }
            if (b < bvalid) {
                int k0 = rev8(t, ndig);
#pragma unroll
                for (int m = 0; m < 8; m++) {
                    if (m < R) {
                        int k = k0 + m * NR;
                        C v = C{a[m].x * scale, a[m].y * sgn * scale};
                        if (PEER) {
                            int pr = k / n_per, kl = k - pr * n_per;
                            peers.p[pr][((int64_t)kl * d_total + outer_start + outer) * n_inner + inner0 + b] = v;
                        } else {
                            dst[outer * outer_stride + inner0 + (int64_t)k * line_stride + b] = v;
                        }
                    }
                }
            }
        }
        __syncthreads();      // the next tile's first stage overwrites the buffer
    }
}

// ---------------------------------------------------------------------------------------------
// Register-I/O line pass with the NEXT tile's first-stage loads in flight during the last stage of the current one
// (ITER first-stage butterflies per thread, Q1 * B == ITER * NT).  With one 512-thread CTA per SM (lines of 1024
// complex doubles) nothing else hides the global-load latency: the loads of tile i+1 are issued before the last stage
// of tile i reads shared memory and streams its outputs out, so the memory system stays busy through the butterflies.
// ---------------------------------------------------------------------------------------------
template <typename T, int B, bool PEER, int NT, int ITER>
__global__ void __launch_bounds__(NT, 512 / NT)
k_fft_lines_rgp(const typename C2<T>::type *src, typename C2<T>::type *dst, PeerPtrs<typename C2<T>::type> peers,
                const typename C2<T>::type *__restrict__ tw, int N, int log2n, int64_t line_stride, int64_t n_inner,
                int64_t tiles_inner, int64_t n_tiles, int64_t outer_stride, int n_per, int64_t d_total,
                int64_t outer_start, int inverse, T scale) {
    typedef typename C2<T>::type C;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    C *sm = reinterpret_cast<C *>(smem_raw);
    constexpr int pitch = B + 1;
    tw = stage_twiddles<C>(sm + (size_t)N * pitch, tw, N);
    const int n8 = log2n / 3, rrem = log2n - 3 * n8;
    const int Q1 = N >> 3;
    const T sgn = inverse ? (T)-1 : (T)1;
    C pre[ITER][8];
    auto issue_loads = [&](int64_t tile) {
        const int64_t outer = tile / tiles_inner;
        const int64_t inner0 = (tile - outer * tiles_inner) * B;
        const C *ibase = src + outer * outer_stride + inner0;
        const int bvalid = (int)((n_inner - inner0) < B ? (n_inner - inner0) : B);
#pragma unroll
        for (int it = 0; it < ITER; it++) {
            const int w = (int)threadIdx.x + it * NT;
            const int b = w % B, q = w / B;
            if (b < bvalid) {
                const C *g = ibase + (int64_t)q * line_stride + b;
#pragma unroll
                for (int j = 0; j < 8; j++) pre[it][j] = g[(int64_t)j * Q1 * line_stride];
            } else {
#pragma unroll
                for (int j = 0; j < 8; j++) pre[it][j] = C{0, 0};
            }
        }
    };
    int64_t tile = blockIdx.x;
    if (tile < n_tiles) issue_loads(tile);
    for (; tile < n_tiles; tile += gridDim.x) {
        const int64_t outer = tile / tiles_inner;
        const int64_t inner0 = (tile - outer * tiles_inner) * B;
        const int bvalid = (int)((n_inner - inner0) < B ? (n_inner - inner0) : B);
        // ---- first stage: registers -> shared
#pragma unroll
        for (int it = 0; it < ITER; it++) {
            const int w = (int)threadIdx.x + it * NT;
            const int b = w % B, q = w / B;
            C a[8];
#pragma unroll
            for (int j = 0; j < 8; j++) { a[j] = pre[it][j]; a[j].y *= sgn; }
            radix8(a);
            C *o = sm + q * pitch + b;
            o[0] = a[0];
#pragma unroll
            for (int m = 1; m < 8; m++) o[m * Q1 * pitch] = cmul(a[m], tw[m * q]);
        }
        __syncthreads();
        // ---- middle stages, in place in shared memory
        {
            const int last8 = rrem ? n8 : n8 - 1;
            int Ns = Q1, lq = log2n - 3;
            for (int s = 1; s < last8; s++) {
                const int Q = Ns >> 3;
                lq -= 3;
                const int tws = N / Ns;
                for (int w = threadIdx.x; w < Q1 * B; w += NT) {
                    int b = w % B, t = w / B;
                    int blk = t >> lq, q = t & (Q - 1);
                    C *p = sm + (blk * Ns + q) * pitch + b;
                    C a[8];
#pragma unroll
                    for (int j = 0; j < 8; j++) a[j] = p[j * Q * pitch];
                    radix8(a);
                    int ti = q * tws;
                    p[0] = a[0];
#pragma unroll
                    for (int m = 1; m < 8; m++) p[m * Q * pitch] = cmul(a[m], tw[m * ti]);
                }
                __syncthreads();
                Ns = Q;
            }
        }
        // ---- the next tile's inputs start travelling now
        if (tile + gridDim.x < n_tiles) issue_loads(tile + gridDim.x);
        // ---- last stage: shared -> registers -> global (frequency rows)
        const int R = rrem == 0 ? 8 : (rrem == 2 ? 4 : 2);
        const int NR = N / R;
        const int ndig = rrem == 0 ? n8 - 1 : n8;
        for (int w = threadIdx.x; w < NR * B; w += NT) {
            int b = w % B, t = w / B;
            const C *p = sm + (t * R) * pitch + b;
            C a[8];
            if (R == 8) {
#pragma unroll
                for (int j = 0; j < 8; j++) a[j] = p[j * pitch];
                radix8(a);
            } else if (R == 4) {
                a[0] = p[0]; a[1] = p[pitch]; a[2] = p[2 * pitch]; a[3] = p[3 * pitch];
                dft4(a[0], a[1], a[2], a[3]);
            } else {
                C x0 = p[0], x1 = p[pitch];
                a[0] = cadd(x0, x1);
                a[1] = csub(x0, x1);
            }
            if (b < bvalid) {
                int k0 = rev8(t, ndig);
#pragma unroll
                for (int m = 0; m < 8; m++) {
                    if (m < R) {
                        int k = k0 + m * NR;
                        C v = C{a[m].x * scale, a[m].y * sgn * scale};
                        if (PEER) {
                            int pr = k / n_per, kl = k - pr * n_per;
                            peers.p[pr][((int64_t)kl * d_total + outer_start + outer) * n_inner + inner0 + b] = v;
                        } else {
                            dst[outer * outer_stride + inner0 + (int64_t)k * line_stride + b] = v;
                        }
                    }
                }
            }
        }
        __syncthreads();      // the next tile's first stage overwrites the buffer
    }
}

// ---------------------------------------------------------------------------------------------
// TMA-pipelined line pass (N = 64 R, R in {4, 8, 16}: lines of 256 / 512 / 1024).  Decimation in TIME over the first
// factor: the line x[n], n = j + R i, splits into R "row groups" j (rows j, j + R, ...: 64 rows of B adjacent columns =
// one 8 KB box of a 4-D tensor map {inner, j, i, outer}), each an independent 64-point FFT, followed by ONE radix-R
// combine  X[k + 64 m] = sum_j W_R^{jm} (W_N^{jk} Y_j[k]).
//   * one elected thread streams the groups of this CTA's tiles through a ring of NS = R + P shared-memory slots with
//     `cp.async.bulk.tensor` (SASS UTMALDG) + one mbarrier per slot: P groups of the NEXT tile are already in flight
//     while this tile is combined, the rest follow as soon as its slots are free -- the copy engine, not the warps'
//     registers, hides the HBM latency, and the warps only run butterflies;
//   * warp w owns group w of the tile: it waits for its own mbarrier and runs the 64-point FFT (8 x 8, two radix-8
//     stages in place, __syncwarp between) while later groups are still landing;
//   * after one CTA barrier every thread combines R values (radix-R in registers, natural output order) and stores the
//     frequency rows k + 64 m straight to global memory (128-byte runs); a second CTA barrier frees the R slots.
// Slots are dense [64][B] with B * sizeof(complex) = 128 bytes, lanes run along the columns first, so every quarter
// warp touches one full 128-byte row: conflict-free without padding.  In place (dst == src) is safe: a tile's stores
// only touch its own rows / columns, which were read completely before its combine.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned fm_smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void fm_mbar_init(uint64_t *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(fm_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fm_mbar_expect_tx(uint64_t *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(fm_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void fm_mbar_wait(uint64_t *bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "NBK_FM_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra NBK_FM_DONE;\n"
        "bra NBK_FM_WAIT;\n"
        "NBK_FM_DONE:\n"
        "}\n" :: "r"(fm_smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void fm_tma_load_4d(void *sdst, const CUtensorMap *tmap, int c0, int c1, int c2, int c3, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
                 :: "r"(fm_smem_u32(sdst)), "l"(tmap), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(fm_smem_u32(bar)) : "memory");
}

template <typename C> struct W16c;      // cos(pi/8), sin(pi/8)
template <> struct W16c<float2> { static __device__ __forceinline__ float c() { return 0.92387953251128675613f; }
                                  static __device__ __forceinline__ float s() { return 0.38268343236508977173f; } };
template <> struct W16c<double2> { static __device__ __forceinline__ double c() { return 0.92387953251128675613; }
                                   static __device__ __forceinline__ double s() { return 0.38268343236508977173; } };

// 16-point forward DFT in registers, natural order in and out (4 x 4: n = 4 n1 + n2, k = k1 + 4 k2)
template <typename C>
__device__ __forceinline__ void dft16(C (&a)[16]) {
    const auto h = Sqrt1_2<C>::v();
    const auto c8 = W16c<C>::c(), s8 = W16c<C>::s();
    C y[4][4];                                   // y[n2][k1]
#pragma unroll
    for (int n2 = 0; n2 < 4; n2++) {
        C b0 = a[n2], b1 = a[4 + n2], b2 = a[8 + n2], b3 = a[12 + n2];
        dft4(b0, b1, b2, b3);
        y[n2][0] = b0; y[n2][1] = b1; y[n2][2] = b2; y[n2][3] = b3;
    }
    // twiddles W_16^{n2 k1}
    y[1][1] = cmul(y[1][1], C{c8, -s8});                                   // W^1
    y[1][2] = C{(y[1][2].x + y[1][2].y) * h, (y[1][2].y - y[1][2].x) * h};  // W^2 = (1 - i)/sqrt2
    y[1][3] = cmul(y[1][3], C{s8, -c8});                                   // W^3
    y[2][1] = C{(y[2][1].x + y[2][1].y) * h, (y[2][1].y - y[2][1].x) * h};  // W^2
    y[2][2] = cmuli_neg(y[2][2]);                                          // W^4 = -i
    y[2][3] = C{(y[2][3].y - y[2][3].x) * h, -(y[2][3].x + y[2][3].y) * h}; // W^6 = (-1 - i)/sqrt2
    y[3][1] = cmul(y[3][1], C{s8, -c8});                                   // W^3
    y[3][2] = C{(y[3][2].y - y[3][2].x) * h, -(y[3][2].x + y[3][2].y) * h}; // W^6
    y[3][3] = cmul(y[3][3], C{-c8, s8});                                   // W^9 = -W^1
#pragma unroll
    for (int k1 = 0; k1 < 4; k1++) {
        C b0 = y[0][k1], b1 = y[1][k1], b2 = y[2][k1], b3 = y[3][k1];
        dft4(b0, b1, b2, b3);
        a[k1] = b0; a[k1 + 4] = b1; a[k1 + 8] = b2; a[k1 + 12] = b3;
    }
}
template <int R, typename C> __device__ __forceinline__ void dftR(C (&a)[R]) {
    if constexpr (R == 16) dft16(a);
    else if constexpr (R == 8) radix8(a);
    else { static_assert(R == 4, "combine radix"); dft4(a[0], a[1], a[2], a[3]); }
}

// CTAs of k_fft_lines_tma per SM, which its shared-memory ring is sized for (2; 3 at N = 256; the tile at N = 1024 takes
// the whole SM).  Also its launch bound: without it ptxas trades spills for an occupancy the ring rules out.
__host__ __device__ constexpr int tma_ctas_per_sm(int R) { return R == 16 ? 1 : R == 4 ? 3 : 2; }

// The 64-point FFTs of a tile's R row groups (warp-local: two radix-8 stages in place); position 8 t + m of a slot
// then holds frequency t + 8 m.  Ends with a CTA barrier.
template <typename T, int R, int B, int NT>
__device__ __forceinline__ void lines_tma_groups(typename C2<T>::type *ring, uint64_t *bars, int NS, int g0,
                                                 const typename C2<T>::type *tw64, T sgn) {
    typedef typename C2<T>::type C;
    constexpr int NW = NT / 32, SLOT = 64 * B;
    static_assert((8 * B) % 32 == 0 && (R % NW == 0 || NW % R == 0), "tile geometry");
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int gw = warp; gw < R; gw += NW) {
        const int g = g0 + gw, slot = g % NS;
        fm_mbar_wait(&bars[slot], (unsigned)((g / NS) & 1));
        C *sl = ring + (size_t)slot * SLOT;
        constexpr int IT = (8 * B) / 32;
#pragma unroll
        for (int i = 0; i < IT; i++) {
            const int w = lane + 32 * i, b = w % B, q = w / B;
            C *p = sl + q * B + b;
            C a[8];
#pragma unroll
            for (int j = 0; j < 8; j++) { a[j] = p[j * 8 * B]; a[j].y *= sgn; }
            radix8(a);
            p[0] = a[0];
#pragma unroll
            for (int m = 1; m < 8; m++) p[m * 8 * B] = cmul(a[m], tw64[m * q]);
        }
        __syncwarp();
#pragma unroll
        for (int i = 0; i < IT; i++) {
            const int w = lane + 32 * i, b = w % B, t = w / B;
            C *p = sl + t * 8 * B + b;
            C a[8];
#pragma unroll
            for (int j = 0; j < 8; j++) a[j] = p[j * B];
            radix8(a);
#pragma unroll
            for (int m = 0; m < 8; m++) p[m * B] = a[m];       // position 8 t + m holds frequency t + 8 m
        }
    }
    __syncthreads();
}

// One tile of the TMA line pass: its R row groups are landing in the ring slots (g0 + j) % NS (g0 = groups this CTA
// streamed before the tile, which also gives each slot's mbarrier phase).  The NT threads run the 64-point FFTs (warp
// w owns groups w, w + NW, ...; warps beyond R wait), the radix-R combine and the stores, then free the R slots: on
// return they may be refilled.
template <typename T, int R, int B, int NT, bool PEER>
__device__ __forceinline__ void lines_tma_tile(typename C2<T>::type *ring, uint64_t *bars, int NS, int g0,
                                               const typename C2<T>::type *twN, const typename C2<T>::type *tw64,
                                               typename C2<T>::type *dst, const PeerPtrs<typename C2<T>::type> &peers,
                                               int64_t line_stride, int64_t n_inner, int64_t outer_stride, int n_per,
                                               int64_t d_total, int64_t outer_start, int64_t outer, int64_t inner0,
                                               T sgn, T scale) {
    typedef typename C2<T>::type C;
    constexpr int S = 64, SLOT = S * B;
    const int tid = threadIdx.x;
    const int bvalid = (int)((n_inner - inner0) < B ? (n_inner - inner0) : B);
    lines_tma_groups<T, R, B, NT>(ring, bars, NS, g0, tw64, sgn);
    // ---- radix-R combine across the groups, registers -> global frequency rows k + 64 m
    {
        const int base = g0 % NS;
        for (int w = tid; w < S * B; w += NT) {
            const int b = w % B, k = w / B;
            const int pos = ((k & 7) << 3) | (k >> 3);
            C a[R];
#pragma unroll
            for (int j = 0; j < R; j++) {
                int sj = base + j;
                if (sj >= NS) sj -= NS;
                C v = ring[(size_t)sj * SLOT + pos * B + b];
                a[j] = j ? cmul(v, twN[j * k]) : v;
            }
            dftR<R, C>(a);
            if (b < bvalid) {
#pragma unroll
                for (int m = 0; m < R; m++) {
                    const int K = k + S * m;
                    const C v = C{a[m].x * scale, a[m].y * sgn * scale};
                    if (PEER) {
                        const int pr = K / n_per, kl = K - pr * n_per;
                        peers.p[pr][((int64_t)kl * d_total + outer_start + outer) * n_inner + inner0 + b] = v;
                    } else {
                        dst[outer * outer_stride + inner0 + (int64_t)K * line_stride + b] = v;
                    }
                }
            }
        }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic accesses to the slots before the next TMA writes
    __syncthreads();
}

template <typename T, int R, int B, int NT, bool PEER>
__global__ void __launch_bounds__(NT, tma_ctas_per_sm(R))
k_fft_lines_tma(const __grid_constant__ CUtensorMap tmap, typename C2<T>::type *dst, PeerPtrs<typename C2<T>::type> peers,
                const typename C2<T>::type *__restrict__ twg, int64_t line_stride, int64_t n_inner, int64_t tiles_inner,
                int64_t n_tiles, int64_t outer_stride, int n_per, int64_t d_total, int64_t outer_start, int inverse, T scale,
                int NS) {
    typedef typename C2<T>::type C;
    // B side-by-side lines: 128-byte rows (8 c16 / 16 c8)
    constexpr int S = 64, N = S * R, SLOT = S * B;
    static_assert(R % (NT / 32) == 0, "tile geometry");
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    C *ring = reinterpret_cast<C *>(smem_raw);                 // [NS][64][B]
    C *twN = ring + (size_t)NS * SLOT;                         // W_N^i, i < N
    C *tw64 = twN + N;                                         // W_64^i, i < 64
    uint64_t *bars = reinterpret_cast<uint64_t *>(tw64 + S);   // [NS]
    const int tid = threadIdx.x;
    if (tid == 0) {
        for (int i = 0; i < NS; i++) fm_mbar_init(&bars[i], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = tid; i < N; i += NT) twN[i] = twg[i];
    for (int i = tid; i < S; i += NT) tw64[i] = twg[i * R];
    __syncthreads();
    const int64_t first = blockIdx.x;
    const int my_tiles = first < n_tiles ? (int)((n_tiles - first + gridDim.x - 1) / gridDim.x) : 0;
    const int G = my_tiles * R;                                // row groups this CTA streams
    const T sgn = inverse ? (T)-1 : (T)1;
    int issued = 0;
    auto issue = [&](int g) {
        const int it = g / R, j = g - it * R;
        const int64_t tile = first + (int64_t)it * gridDim.x;
        const int64_t outer = tile / tiles_inner;
        const int64_t inner0 = (tile - outer * tiles_inner) * B;
        const int slot = g % NS;
        fm_mbar_expect_tx(&bars[slot], (unsigned)(SLOT * sizeof(C)));
        fm_tma_load_4d(ring + (size_t)slot * SLOT, &tmap, (int)(2 * inner0), j, 0, (int)outer, &bars[slot]);
    };
    if (tid == 0) {
        const int upto = G < NS ? G : NS;
        for (; issued < upto; issued++) issue(issued);
    }
    for (int it = 0; it < my_tiles; it++) {
        const int64_t tile = first + (int64_t)it * gridDim.x;
        const int64_t outer = tile / tiles_inner;
        const int64_t inner0 = (tile - outer * tiles_inner) * B;
        lines_tma_tile<T, R, B, NT, PEER>(ring, bars, NS, it * R, twN, tw64, dst, peers, line_stride, n_inner,
                                          outer_stride, n_per, d_total, outer_start, outer, inner0, sgn, scale);
        if (tid == 0) {
            int upto = (it + 1) * R + NS;
            if (upto > G) upto = G;
            for (; issued < upto; issued++) issue(issued);
        }
    }
}

typedef CUresult (*nbk_encode_tiled_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                        const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static nbk_encode_tiled_fn get_tensor_map_encoder() {
    static std::mutex m;
    static bool tried = false;
    static nbk_encode_tiled_fn fn = nullptr;
    std::lock_guard<std::mutex> lock(m);
    if (!tried) {
        tried = true;
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (nbk_encode_tiled_fn)p;
        else
            (void)cudaGetLastError();
    }
    return fn;
}

// ---------------------------------------------------------------------------------------------
// z pass forward: real rows [rows][Nz] -> complex rows [rows][Nz/2+1]
// packed trick: z[n] = x[2n] + i x[2n+1], Z = FFT_M(z), M = Nz/2,
//   X[k] = 1/2 [ (Z[k] + conj Z[M-k]) - i W_N^k (Z[k] - conj Z[M-k]) ],  k = 0..M  (Z[M] := Z[0])
// ---------------------------------------------------------------------------------------------
template <typename T, int B>
__global__ void __launch_bounds__(256)
k_fft_z_r2c(const T *__restrict__ real, typename C2<T>::type *__restrict__ cplx,
            const typename C2<T>::type *__restrict__ twM, const typename C2<T>::type *__restrict__ twN, int Nz,
            int log2m, int64_t rows, T scale) {
    typedef typename C2<T>::type C;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    C *sm = reinterpret_cast<C *>(smem_raw);
    const int M = Nz >> 1;
    const int Nzc = M + 1;
    constexpr int pitch = B + 1;
    const int T_ = blockDim.x;
    const int sk = log2m >= 3 ? log2m - 3 : 31;
    const int64_t n_tiles = (rows + B - 1) / B;
    twM = stage_twiddles<C>(sm + M * pitch + 8, twM, M);
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        int64_t row0 = tile * B;
        int bvalid = (int)((rows - row0) < B ? (rows - row0) : B);
        const C *src = reinterpret_cast<const C *>(real + row0 * Nz);  // rows of M packed pairs, 2*sizeof(T) aligned
        for (int w = threadIdx.x; w < M * B; w += T_) {
            int n = w & (M - 1), b = w >> log2m;  // lanes run along the contiguous row
            C v = C{0, 0};
            if (b < bvalid) v = src[(int64_t)b * M + n];
            sm[saddr<B, true>(n, sk) + b] = v;
        }
        __syncthreads();
        fft_tile<C, B, true>(sm, twM, M, log2m);
        C *dst = cplx + row0 * Nzc;
        for (int w = threadIdx.x; w < Nzc * B; w += T_) {
            int k = w % Nzc, b = w / Nzc;
            if (b < bvalid) {
                C zk = sm[saddr<B, true>(pos_of_freq(k & (M - 1), M, log2m), sk) + b];
                C zm = cconj(sm[saddr<B, true>(pos_of_freq((M - k) & (M - 1), M, log2m), sk) + b]);
                C e = cadd(zk, zm), o = csub(zk, zm);
                C wo = cmul(twN[k], o);          // W_N^k (Z[k] - conj Z[M-k])
                C x = C{e.x + wo.y, e.y - wo.x};  // e - i*wo
                T h = (T)0.5 * scale;
                dst[(int64_t)b * Nzc + k] = C{x.x * h, x.y * h};
            }
        }
        __syncthreads();
    }
}

// Last DIF stage of B side-by-side length-M lines in shared memory, leaving the spectrum in NATURAL order: every thread
// first pulls all of its butterflies into registers (V values: M * B <= 256 V; V = 16 for c8, 8 for c16 keeps them in 32 registers), then the CTA
// synchronises, then the outputs are stored at their frequency rows.
template <typename C, int B, int R, int V>
__device__ __forceinline__ void last_stage_natural(C *sm, int M, int ndig) {
    constexpr int pitch = B + 1;
    constexpr int NB = V / R;
    const int NR = M / R;
    C a[NB][R];
#pragma unroll
    for (int it = 0; it < NB; it++) {
        int w = threadIdx.x + it * 256;
        if (w < NR * B) {
            int b = w % B, t = w / B;
            const C *p = sm + (t * R) * pitch + b;
#pragma unroll
            for (int j = 0; j < R; j++) a[it][j] = p[j * pitch];
            if constexpr (R == 8) {
                radix8(a[it]);
            } else if constexpr (R == 4) {
                dft4(a[it][0], a[it][1], a[it][2], a[it][3]);
            } else {
                C x0 = a[it][0], x1 = a[it][1];
                a[it][0] = cadd(x0, x1);
                a[it][1] = csub(x0, x1);
            }
        }
    }
    __syncthreads();
#pragma unroll
    for (int it = 0; it < NB; it++) {
        int w = threadIdx.x + it * 256;
        if (w < NR * B) {
            int b = w % B, t = w / B;
            int k0 = rev8(t, ndig);
#pragma unroll
            for (int m = 0; m < R; m++) sm[(k0 + m * NR) * pitch + b] = a[it][m];
        }
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// z pass forward, register-I/O variant (Nz >= 128).  Same packed-pair algorithm as k_fft_z_r2c; the first radix-8
// stage reads the real row straight from global memory (lanes along the row: 512-byte runs), the last stage leaves
// Z in NATURAL frequency order in shared memory (registers carry the permutation across one barrier), so the
// Hermitian split reads Z[k] and Z[M-k] with unit-stride lanes and no digit-reversal arithmetic.  Shared: tile
// [M][B+1] | W_N table [N] (W_M^j = W_N^2j serves the butterflies, W_N^k the split) | first-stage twiddles [7][M/8].
// ---------------------------------------------------------------------------------------------
template <typename T, int B>
__global__ void __launch_bounds__(256, 2)
k_fft_z_r2c_rg(const T *__restrict__ real, typename C2<T>::type *__restrict__ cplx,
               const typename C2<T>::type *__restrict__ twN_g, int Nz, int log2m, int64_t rows, T scale) {
    typedef typename C2<T>::type C;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    C *sm = reinterpret_cast<C *>(smem_raw);
    const int M = Nz >> 1;
    const int Nzc = M + 1;
    constexpr int pitch = B + 1;
    const int T_ = blockDim.x;
    // first-stage twiddles transposed to [m][q] (lanes run along q there: unit stride instead of stride 2m)
    C *tw1 = sm + (size_t)M * pitch + Nz;
    for (int i = threadIdx.x; i < 7 * (M >> 3); i += blockDim.x) {
        int m = i / (M >> 3) + 1, q = i - (m - 1) * (M >> 3);
        tw1[i] = twN_g[2 * m * q];
    }
    const C *tw = stage_twiddles<C>(sm + (size_t)M * pitch, twN_g, Nz);    // tw[2j] = W_M^j
    const int n8 = log2m / 3, rrem = log2m - 3 * n8;
    const int Q1 = M >> 3, lq1 = log2m - 3;
    const int64_t n_tiles = (rows + B - 1) / B;
    const T h = (T)0.5 * scale;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t row0 = tile * B;
        const int bvalid = (int)((rows - row0) < B ? (rows - row0) : B);
        const C *src = reinterpret_cast<const C *>(real + row0 * Nz);    // rows of M packed pairs
        // ---- first stage: global -> registers -> shared; lanes along the row
        for (int w = threadIdx.x; w < Q1 * B; w += T_) {
            int q = w & (Q1 - 1), b = w >> lq1;
            C a[8];
            if (b < bvalid) {
                const C *g = src + (int64_t)b * M + q;
#pragma unroll
                for (int j = 0; j < 8; j++) a[j] = g[j * Q1];
            } else {
#pragma unroll
                for (int j = 0; j < 8; j++) a[j] = C{0, 0};
            }
            radix8(a);
            C *o = sm + q * pitch + b;
            o[0] = a[0];
#pragma unroll
            for (int m = 1; m < 8; m++) o[m * Q1 * pitch] = cmul(a[m], tw1[(m - 1) * Q1 + q]);
        }
        __syncthreads();
        // ---- middle stages, in place
        {
            const int last8 = rrem ? n8 : n8 - 1;
            int Ns = Q1, lq = lq1;
            for (int s = 1; s < last8; s++) {
                const int Q = Ns >> 3;
                lq -= 3;
                const int tws = 2 * (M / Ns);
                for (int w = threadIdx.x; w < Q1 * B; w += T_) {
                    int b = w % B, t = w / B;
                    int blk = t >> lq, q = t & (Q - 1);
                    C *p = sm + (blk * Ns + q) * pitch + b;
                    C a[8];
#pragma unroll
                    for (int j = 0; j < 8; j++) a[j] = p[j * Q * pitch];
                    radix8(a);
                    int ti = q * tws;
                    p[0] = a[0];
#pragma unroll
                    for (int m = 1; m < 8; m++) p[m * Q * pitch] = cmul(a[m], tw[m * ti]);
                }
                __syncthreads();
                Ns = Q;
            }
        }
        // ---- last stage: all M*B/256 <= V values of a thread go to registers, barrier, natural-order write back
        constexpr int V = sizeof(T) == 4 ? 16 : 8;
        if (rrem == 0) last_stage_natural<C, B, 8, V>(sm, M, n8 - 1);
        else if (rrem == 2) last_stage_natural<C, B, 4, V>(sm, M, n8);
        else last_stage_natural<C, B, 2, V>(sm, M, n8);
        // ---- Hermitian split, one warp per row, lanes along k
        C *dst = cplx + row0 * Nzc;
        for (int b = threadIdx.x >> 5; b < bvalid; b += (T_ >> 5)) {
            C *drow = dst + (int64_t)b * Nzc;
            for (int k = threadIdx.x & 31; k < Nzc; k += 32) {
                C zk = sm[(k & (M - 1)) * pitch + b];
                C zm = cconj(sm[((M - k) & (M - 1)) * pitch + b]);
                C e = cadd(zk, zm), o = csub(zk, zm);
                C wo = cmul(tw[k], o);
                drow[k] = C{(e.x + wo.y) * h, (e.y - wo.x) * h};
            }
        }
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------
// z pass forward, warp-per-row with TMA bulk row copies (Nz = 2M, M in {128, 256, 512}).  Every warp owns a private ring of
// row buffers: one lane streams the next rows of the warp in with `cp.async.bulk` (one 1-D copy of the whole row, SASS
// UBLKCP) + an mbarrier per buffer while the warp transforms the row that has landed -- packed-pair M-point FFT (radix 8,
// 8, M/64, in place, __syncwarp between the stages), Hermitian split, coalesced stores of the Nz/2+1 modes.  No CTA
// barrier after the twiddle staging, so the warps of an SM drift apart and the loads never stop.
// Shared-memory positions are XOR-swizzled, pos(e) = e ^ ((e >> 3) & 7) (a permutation inside each aligned group of 8
// elements = one 128-byte line of c16), which makes the stride-8 accesses of the later stages and the natural-order
// write of the last stage bank-conflict free; the copy engine lands the row unswizzled and the first stage re-places it.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void fm_bulk_g2s(void *sdst, const void *gsrc, unsigned bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(fm_smem_u32(sdst)), "l"(gsrc), "r"(bytes), "r"(fm_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ int fm_sw(int e) { return e ^ ((e >> 3) & 7); }

// L2 policies for the pipelined z + y pass (k_fft_zy_r2c_pipe): its z stores ask L2 to keep their lines for the y
// tiles that read them back, and its reads of the real field, used once, ask to leave first.
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void st_hint(double2 *p, double2 v, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.v2.f64 [%0], {%1, %2}, %3;" :: "l"(p), "d"(v.x), "d"(v.y), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_hint(float2 *p, float2 v, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.v2.f32 [%0], {%1, %2}, %3;" :: "l"(p), "f"(v.x), "f"(v.y), "l"(pol) : "memory");
}
__device__ __forceinline__ void fm_bulk_g2s_hint(void *sdst, const void *gsrc, unsigned bytes, uint64_t *bar, uint64_t pol) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 :: "r"(fm_smem_u32(sdst)), "l"(gsrc), "r"(bytes), "r"(fm_smem_u32(bar)), "l"(pol) : "memory");
}

// Twiddle tables of the warp-per-row z pass in shared memory: W_N^i, i < Nz (Hermitian split) | [7][Q1] W_M^{q m},
// lanes along q at unit stride | [7][8] W_{8 R3}^{q m}.  All threads of the CTA call; a CTA barrier must follow.
template <typename C, int LM, int NT>
__device__ __forceinline__ void z_r2c_stage_twiddles(C *twN, const C *__restrict__ twN_g) {
    constexpr int M = 1 << LM, Nz = 2 * M, R3 = M / 64, Q1 = M / 8;
    C *tw1 = twN + Nz, *tw2 = tw1 + 7 * Q1;
    for (int i = threadIdx.x; i < Nz; i += NT) twN[i] = twN_g[i];
    // (a strided twN[2 m q] / twN[16 m q] puts the lanes of a quarter warp on the same banks: 8-way conflicts that made
    // the twiddle reads cost more shared-memory wavefronts than the data)
    for (int i = threadIdx.x; i < 7 * Q1; i += NT) { const int m = i / Q1 + 1, q = i % Q1; tw1[i] = twN_g[2 * m * q]; }
    for (int i = threadIdx.x; i < 7 * R3; i += NT) { const int m = i / R3 + 1, q = i % R3; tw2[i] = twN_g[(16 * m * q) % Nz]; }
}
template <int LM> __host__ __device__ constexpr int z_r2c_twiddle_len() { return 2 * (1 << LM) + 7 * ((1 << LM) / 8) + 7 * 8; }

// One warp transforms n real rows, row i = first + i * stride (i < n), streaming them through its private ring of nbuf
// row buffers (wbuf [nbuf][M], one mbarrier each in wbar).  c0 = rows the warp streamed through the ring before: slots
// and mbarrier phases continue from there.  KEEP: the real rows are read with an L2 evict-first hint and the complex
// rows stored with an evict-last one (the pipelined z + y pass); otherwise plain loads and stores.
template <typename T, int LM, bool KEEP>
__device__ __forceinline__ void z_r2c_warp_rows(const T *__restrict__ real, typename C2<T>::type *__restrict__ cplx,
                                                const typename C2<T>::type *twN, typename C2<T>::type *wbuf,
                                                uint64_t *wbar, int nbuf, int64_t c0, int64_t first, int64_t stride,
                                                int64_t n, T h) {
    typedef typename C2<T>::type C;
    constexpr int M = 1 << LM, Nz = 2 * M, Nzc = M + 1;
    constexpr int R3 = M / 64;                    // last radix: 8 / 4 / 2
    constexpr int Q1 = M / 8;                     // butterflies of the radix-8 stages
    constexpr int I1 = (Q1 + 31) / 32;            // ... per lane
    const C *tw1 = twN + Nz, *tw2 = tw1 + 7 * Q1;
    // read here (volatile): in the persistent k_fft_zy_r2c_pipe the per-lane shared addresses would otherwise be hoisted
    // out of its work loop, held across the y tiles, and spilled
    int lane;
    asm volatile("mov.u32 %0, %%laneid;" : "=r"(lane));
    lane &= 31;
    const unsigned row_bytes = (unsigned)(M * sizeof(C));
    uint64_t pol_in = 0, pol_out = 0;
    if (KEEP) { pol_in = l2_policy_evict_first(); pol_out = l2_policy_evict_last(); }
    auto issue = [&](int64_t i) {     // lane 0 only
        const int sidx = (int)((c0 + i) % nbuf);
        fm_mbar_expect_tx(&wbar[sidx], row_bytes);
        const T *src = real + (first + i * stride) * (int64_t)Nz;
        if (KEEP) fm_bulk_g2s_hint(wbuf + (size_t)sidx * M, src, row_bytes, &wbar[sidx], pol_in);
        else fm_bulk_g2s(wbuf + (size_t)sidx * M, src, row_bytes, &wbar[sidx]);
    };
    if (lane == 0) for (int64_t i = 0; i < nbuf && i < n; i++) issue(i);
    for (int64_t i = 0; i < n; i++) {
        const int sidx = (int)((c0 + i) % nbuf);
        fm_mbar_wait(&wbar[sidx], (unsigned)(((c0 + i) / nbuf) & 1));
        C *z = wbuf + (size_t)sidx * M;
        // ---- stage 1 (radix 8 over elements q + Q1 j): reads the landed (unswizzled) row, writes swizzled
        {
            C a[I1][8];
#pragma unroll
            for (int it = 0; it < I1; it++) {
                const int q = lane + 32 * it;
                if (q < Q1) {
#pragma unroll
                    for (int j = 0; j < 8; j++) a[it][j] = z[q + Q1 * j];
                }
            }
            __syncwarp();
#pragma unroll
            for (int it = 0; it < I1; it++) {
                const int q = lane + 32 * it;
                if (q < Q1) {
                    radix8(a[it]);
                    z[fm_sw(q)] = a[it][0];
#pragma unroll
                    for (int m = 1; m < 8; m++) z[fm_sw(q + Q1 * m)] = cmul(a[it][m], tw1[(m - 1) * Q1 + q]);
                }
            }
        }
        __syncwarp();
        // ---- stage 2 (radix 8 inside the 8 blocks of Q1 elements: elements blk Q1 + q + R3 j), in place
#pragma unroll
        for (int it = 0; it < I1; it++) {
            const int t = lane + 32 * it;
            if (t < Q1) {
                const int blk = t / R3, q = t - blk * R3;
                const int e0 = blk * Q1 + q;
                C a[8];
#pragma unroll
                for (int j = 0; j < 8; j++) a[j] = z[fm_sw(e0 + R3 * j)];
                radix8(a);
                z[fm_sw(e0)] = a[0];
#pragma unroll
                for (int m = 1; m < 8; m++) z[fm_sw(e0 + R3 * m)] = cmul(a[m], tw2[(m - 1) * R3 + q]);      // W_{8 R3}^{q m}
            }
        }
        __syncwarp();
        // ---- stage 3 (radix R3 over elements R3 t + j, 64 butterflies); outputs go to NATURAL frequency positions:
        // position R3 t + m3 holds frequency (t / 8) + 8 (t % 8) + 64 m3
        {
            C a[2][R3];
#pragma unroll
            for (int it = 0; it < 2; it++) {
                const int t = lane + 32 * it;
#pragma unroll
                for (int j = 0; j < R3; j++) a[it][j] = z[fm_sw(R3 * t + j)];
            }
            __syncwarp();
#pragma unroll
            for (int it = 0; it < 2; it++) {
                const int t = lane + 32 * it;
                if constexpr (R3 == 8) radix8(a[it]);
                else if constexpr (R3 == 4) dft4(a[it][0], a[it][1], a[it][2], a[it][3]);
                else { C x0 = a[it][0], x1 = a[it][1]; a[it][0] = cadd(x0, x1); a[it][1] = csub(x0, x1); }
                const int k0 = (t >> 3) + 8 * (t & 7);
#pragma unroll
                for (int m = 0; m < R3; m++) z[fm_sw(k0 + 64 * m)] = a[it][m];
            }
        }
        __syncwarp();
        // ---- Hermitian split, lanes along k:  X[k] = 1/2 [ (Z[k] + conj Z[M-k]) - i W_N^k (Z[k] - conj Z[M-k]) ]
        C *drow = cplx + (first + i * stride) * (int64_t)Nzc;
        for (int k = lane; k < Nzc; k += 32) {
            const C zk = z[fm_sw(k & (M - 1))];
            const C zm = cconj(z[fm_sw((M - k) & (M - 1))]);
            const C e = cadd(zk, zm), o = csub(zk, zm);
            const C wo = cmul(twN[k], o);
            const C v = C{(e.x + wo.y) * h, (e.y - wo.x) * h};
            if (KEEP) st_hint(drow + k, v, pol_out);
            else drow[k] = v;
        }
        // ---- the buffer is free: fetch the row that will use it next
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        if (lane == 0 && i + nbuf < n) issue(i + nbuf);
    }
}

template <typename T, int LM, int NW>
__global__ void __launch_bounds__(32 * NW)
k_fft_z_r2c_tma(const T *__restrict__ real, typename C2<T>::type *__restrict__ cplx,
                const typename C2<T>::type *__restrict__ twN_g, int64_t rows, T scale, int nbuf) {
    typedef typename C2<T>::type C;
    constexpr int M = 1 << LM;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    C *twN = reinterpret_cast<C *>(smem_raw);                         // twiddle tables (z_r2c_stage_twiddles)
    C *bufs = twN + z_r2c_twiddle_len<LM>();                          // [NW][nbuf][M]
    uint64_t *bars = reinterpret_cast<uint64_t *>(bufs + (size_t)NW * nbuf * M);   // [NW][nbuf]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    z_r2c_stage_twiddles<C, LM, 32 * NW>(twN, twN_g);
    if (lane == 0) {
        for (int i = 0; i < nbuf; i++) fm_mbar_init(&bars[warp * nbuf + i], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int64_t gw = (int64_t)blockIdx.x * NW + warp, GW = (int64_t)gridDim.x * NW;
    const int64_t my_rows = gw < rows ? (rows - gw + GW - 1) / GW : 0;
    z_r2c_warp_rows<T, LM, false>(real, cplx, twN, bufs + (size_t)warp * nbuf * M, bars + warp * nbuf, nbuf, 0, gw, GW,
                                  my_rows, (T)0.5 * scale);
}

// ---------------------------------------------------------------------------------------------
// Forward z + y passes of the power-of-two r2c, pipelined plane by plane (Nz = 2M, M in {128, 256, 512}; Ny = 64 R,
// R in {4, 8, 16}; c16 fields).  Run one after the other, the z pass writes the whole half spectrum to HBM and the y
// pass reads it straight back.  Here the y tiles of an x plane run shortly after that plane's z rows, so they read the
// rows from L2, and their in-place stores overwrite lines that are still dirty there: each complex plane reaches DRAM
// once (4 field-sizes of DRAM traffic for the r2c instead of 6).  The arithmetic is that of the two separate passes
// (the same device functions, k_fft_z_r2c_tma's rows and k_fft_lines_tma's tiles): the result is bit-identical.
//   * persistent CTAs of 512 threads take tickets from one global counter.  Ticket t is item t % L of step t / L, where
//     a step lists the NZI z items of plane t / L (ZROWS rows each, warp-per-row) and then the NYI y tiles of plane
//     t / L - D (B columns over all Ny rows); items of planes outside [0, x_n) are skipped;
//   * a z item stamps its flag with this call's epoch once its rows are stored; a y tile polls the NZI flags of its
//     plane (relaxed loads, then an acquire fence) and sleeps while any is older than the epoch;
//   * deadlock-free by construction: a y tile waits only on z items of lower tickets, every one of which has been
//     taken by a running CTA that never waits (z items wait on nothing), so the lowest unfinished ticket always makes
//     progress -- whatever the grid size and however many CTAs are resident;
//   * the ticket counter returns to 0 at the end of every call: every CTA takes tickets until one is past the last item,
//     so exactly n_items + gridDim.x tickets are taken, and the CTA that takes the last one resets the counter.  The
//     counter and the flags belong to the calling stream (ZyPipeSync): calls on other streams never touch them;
//   * z and y items share the dynamic shared memory (z row buffers | y ring slots); each item drains its own copies
//     before it returns, so the next item, of either kind, starts on free buffers.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned ld_relaxed_gpu(const unsigned *p) {
    unsigned v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_gpu(unsigned *p, unsigned v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}

// threads of the pipelined z + y pass; rows per warp in one z item; complex values of each warp's z ring (its nbuf =
// ZY_ZBUF / M row buffers: 1 / 2 / 4 at M = 512 / 256 / 128 fill the 128 KB a y tile of 1024-point lines takes)
constexpr int ZY_NT = 512, ZY_ZPW = 2, ZY_ZBUF = 512;

template <typename T, int LM, int R>
__global__ void __launch_bounds__(ZY_NT, 1)
k_fft_zy_r2c_pipe(const __grid_constant__ CUtensorMap tmap, const T *__restrict__ real, typename C2<T>::type *cplx,
                  const typename C2<T>::type *__restrict__ twz_g, const typename C2<T>::type *__restrict__ twy_g,
                  int x_n, int D, unsigned *ticket, unsigned *flags, unsigned epoch, T scale, T sgn) {
    typedef typename C2<T>::type C;
    constexpr int NT = ZY_NT, NW = NT / 32, M = 1 << LM, Nzc = M + 1, S = 64, Ny = S * R;
    constexpr int B = 128 / (int)sizeof(C), SLOT = S * B;
    constexpr int ZROWS = NW * ZY_ZPW;
    constexpr int NZI = Ny / ZROWS, NYI = (Nzc + B - 1) / B, L = NZI + NYI;
    constexpr int nbuf = ZY_ZBUF / M, NS = R;                // z ring: ZY_ZBUF complex per warp; y ring: one tile
    static_assert(NZI <= 32, "one lane polls one z flag");
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    constexpr size_t zbuf = (size_t)NW * nbuf * M, ybuf = (size_t)NS * SLOT;
    C *ring = reinterpret_cast<C *>(smem_raw);                 // z row buffers [NW][nbuf][M] | y slots [NS][64][B]
    C *twz = ring + (zbuf > ybuf ? zbuf : ybuf);                // z twiddle tables (z_r2c_stage_twiddles)
    C *twy = twz + z_r2c_twiddle_len<LM>();                    // W_Ny^i, i < Ny
    C *tw64 = twy + Ny;                                        // W_64^i, i < 64
    uint64_t *zbars = reinterpret_cast<uint64_t *>(tw64 + S);  // [NW][nbuf]
    uint64_t *ybars = zbars + NW * nbuf;                       // [NS]
    unsigned *s_ticket = reinterpret_cast<unsigned *>(ybars + NS);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    z_r2c_stage_twiddles<C, LM, NT>(twz, twz_g);
    for (int i = tid; i < Ny; i += NT) twy[i] = twy_g[i];
    for (int i = tid; i < S; i += NT) tw64[i] = twy_g[i * R];
    if (tid == 0) {
        for (int i = 0; i < NW * nbuf; i++) fm_mbar_init(&zbars[i], 1);
        for (int i = 0; i < NS; i++) fm_mbar_init(&ybars[i], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const PeerPtrs<C> no_peers{};
    const unsigned n_items = (unsigned)L * (unsigned)(x_n + D);
    const T h = (T)0.5 * scale;
    int zc = 0;                 // rows each warp has streamed through its z ring
    int yc = 0;                 // row groups the CTA has streamed through the y ring
    for (;;) {
        if (tid == 0) {
            const unsigned t = atomicAdd(ticket, 1u);
            if (t == n_items + gridDim.x - 1) atomicExch(ticket, 0u);
            *s_ticket = t;
        }
        __syncthreads();
        const unsigned t = *s_ticket;
        __syncthreads();
        if (t >= n_items) break;
        const int step = (int)(t / L), r = (int)(t % L);
        if (r < NZI) {
            const int p = step;
            if (p >= x_n) continue;
            const int64_t row0 = (int64_t)p * Ny + (int64_t)r * ZROWS;
            z_r2c_warp_rows<T, LM, true>(real, cplx, twz, ring + (size_t)warp * nbuf * M, zbars + warp * nbuf, nbuf, zc,
                                         row0 + warp, NW, ZY_ZPW, h);
            zc += ZY_ZPW;
            asm volatile("fence.proxy.async.global;" ::: "memory");   // the rows are read back through the copy engine
            __syncthreads();
            if (tid == 0) st_release_gpu(&flags[(int64_t)p * NZI + r], epoch);   // cumulative over the CTA's stores
        } else {
            const int q = step - D;
            if (q < 0) continue;
            const int64_t inner0 = (int64_t)(r - NZI) * B;
            if (warp == 0) {
                if (lane < NZI) {
                    const unsigned *f = flags + (int64_t)q * NZI + lane;
                    while (ld_relaxed_gpu(f) < epoch) __nanosleep(256);
                    asm volatile("fence.acq_rel.gpu;" ::: "memory");
                }
                __syncwarp();
                if (lane == 0) {
                    asm volatile("fence.proxy.async.global;" ::: "memory");
                    for (int j = 0; j < R; j++) {
                        const int slot = (yc + j) % NS;
                        fm_mbar_expect_tx(&ybars[slot], (unsigned)(SLOT * sizeof(C)));
                        fm_tma_load_4d(ring + (size_t)slot * SLOT, &tmap, (int)(2 * inner0), j, 0, q, &ybars[slot]);
                    }
                }
            }
            lines_tma_tile<T, R, B, NT, false>(ring, ybars, NS, yc, twy, tw64, cplx, no_peers, Nzc, Nzc,
                                               (int64_t)Ny * Nzc, Ny, 0, 0, q, inner0, sgn, scale);
            yc += R;
        }
    }
}

// z pass backward: complex rows [rows][Nz/2+1] -> real rows [rows][Nz], unnormalised
//   E = (X[k] + conj X[M-k])/2, O = conj(W_N^k) (X[k] - conj X[M-k])/2, Z[k] = E + i O, k < M
//   x[2n] + i x[2n+1] = 2 * sum_k Z[k] e^{+2 pi i k n / M} = 2 * conj(FFT_M(conj Z))[n]
template <typename T, int B>
__global__ void __launch_bounds__(256)
k_fft_z_c2r(const typename C2<T>::type *__restrict__ cplx, T *__restrict__ real,
            const typename C2<T>::type *__restrict__ twM, const typename C2<T>::type *__restrict__ twN, int Nz,
            int log2m, int64_t rows) {
    typedef typename C2<T>::type C;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    C *sm = reinterpret_cast<C *>(smem_raw);
    const int M = Nz >> 1;
    const int Nzc = M + 1;
    constexpr int pitch = B + 1;
    const int T_ = blockDim.x;
    const int sk = log2m >= 3 ? log2m - 3 : 31;
    const int64_t n_tiles = (rows + B - 1) / B;
    twM = stage_twiddles<C>(sm + M * pitch + 8, twM, M);
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        int64_t row0 = tile * B;
        int bvalid = (int)((rows - row0) < B ? (rows - row0) : B);
        const C *src = cplx + row0 * Nzc;
        for (int w = threadIdx.x; w < M * B; w += T_) {
            int k = w & (M - 1), b = w >> log2m;
            C v = C{0, 0};
            if (b < bvalid) {
                C xk = src[(int64_t)b * Nzc + k];
                C xm = cconj(src[(int64_t)b * Nzc + (M - k)]);
                if (k == 0) { xk.y = 0; xm.y = 0; }     // the k = 0 and k = Nz/2 modes of a real row are real
                C e = cadd(xk, xm), d = csub(xk, xm);
                C o = cmul(cconj(twN[k]), d);
                // Z = (e + i o)/2 ; the factor 2 of the unnormalised inverse cancels the 1/2
                C z = C{e.x - o.y, e.y + o.x};
                v = cconj(z);
            }
            sm[saddr<B, true>(k, sk) + b] = v;
        }
        __syncthreads();
        fft_tile<C, B, true>(sm, twM, M, log2m);
        C *dst = reinterpret_cast<C *>(real + row0 * Nz);
        for (int w = threadIdx.x; w < M * B; w += T_) {
            int n = w & (M - 1), b = w >> log2m;
            if (b < bvalid) {
                C v = cconj(sm[saddr<B, true>(pos_of_freq(n, M, log2m), sk) + b]);
                dst[(int64_t)b * M + n] = v;
            }
        }
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------
// twiddle tables, cached per (device, N, dtype)
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void k_twiddle(typename C2<T>::type *tw, int N) {
    int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < N) {
        double s, c;
        sincospi(-2.0 * (double)k / (double)N, &s, &c);
        tw[k].x = (T)c;
        tw[k].y = (T)s;
    }
}

static std::mutex g_tw_mutex;
static std::map<std::tuple<int, int, int>, void *> g_tw;

static int get_twiddle(int N, int dtype, cudaStream_t s, void **out) {
    int dev = 0;
    NBK_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(g_tw_mutex);
    auto key = std::make_tuple(dev, N, dtype);
    auto it = g_tw.find(key);
    if (it != g_tw.end()) { *out = it->second; return NBK_OK; }
    void *p = nullptr;
    size_t bytes = (size_t)(N > 0 ? N : 1) * (dtype == NBK_F4 ? 8 : 16);
    NBK_CUDA(cudaMalloc(&p, bytes));
    int g = (N + 255) / 256;
    if (g < 1) g = 1;
    if (dtype == NBK_F4) k_twiddle<float><<<g, 256, 0, s>>>((float2 *)p, N);
    else k_twiddle<double><<<g, 256, 0, s>>>((double2 *)p, N);
    NBK_LAUNCHED();
    // table must be visible to later launches on other streams as well
    NBK_CUDA(cudaStreamSynchronize(s));
    g_tw[key] = p;
    *out = p;
    return NBK_OK;
}

static int ilog2(int64_t n) {
    int l = 0;
    while (((int64_t)1 << l) < n) l++;
    return l;
}
static bool is_pow2(int64_t n) { return n > 0 && (n & (n - 1)) == 0; }
// longest power-of-two complex line (x / y lines; the z pass runs Nz/2-point lines): one CTA keeps a whole line of
// at least N (B + 2) complex values, B >= 1, in its 227 KB of shared memory -- 8192 points in f4, 4096 in f8
static int64_t pow2_max_line(int dtype) { return dtype == NBK_F4 ? 8192 : 4096; }

// pick the number of side-by-side lines: >= 64 B contiguous runs, tile <= ~96 KB (2 CTAs / SM)
static int pick_B(int N, int csize, int64_t n_inner) {
    int B = 128 / csize;  // 128-byte runs: 16 (c8) or 8 (c16)
    while (B > 1 && (size_t)N * (B + 2) * csize > 98304) B >>= 1;
    while (B > 1 && B / 2 >= n_inner) B >>= 1;
    return B;
}

// TMA-pipelined line pass (k_fft_lines_tma) where it applies: N in {256, 512, 1024}, 16-byte aligned rows (always true
// for c16 fields; c8 fields with an odd row length -- the y pass over Nz/2+1 columns -- keep the register-I/O kernel).
// *done = false: not applicable, the caller falls back.  d_total: rows of the peer field (peer stores only).
// Tensor map of the TMA line pass over lines of N = 64 R complex values: 4-D {inner (as 2 n_inner reals), j, i, outer}
// with line element n = j + R i, boxes of one row group (64 rows of B = 128 / sizeof(complex) columns).  false: the
// shape does not qualify (unaligned rows, out of the encoder's range, no encoder): the caller keeps the older kernels.
template <typename T>
static bool encode_lines_tmap(CUtensorMap *tmap, const void *src, int N, int64_t line_stride, int64_t n_inner,
                              int64_t n_outer, int64_t ostride) {
    typedef typename C2<T>::type C;
    const size_t cs = sizeof(C);
    if ((reinterpret_cast<uintptr_t>(src) & 15) || ((size_t)line_stride * cs) % 16 || ((size_t)ostride * cs) % 16) return false;
    if (2 * n_inner >= (1ll << 31) || n_outer >= (1ll << 31) || (size_t)ostride * cs >= ((size_t)1 << 40) ||
        (size_t)(N / 64) * line_stride * cs >= ((size_t)1 << 40)) return false;
    nbk_encode_tiled_fn enc = get_tensor_map_encoder();
    if (!enc) return false;
    const int R = N / 64;
    constexpr int B = 128 / (int)sizeof(C);                    // tile width: 128-byte rows
    const cuuint64_t gdim[4] = {(cuuint64_t)(2 * n_inner), (cuuint64_t)R, 64, (cuuint64_t)n_outer};
    const cuuint64_t gstr[3] = {(cuuint64_t)line_stride * cs, (cuuint64_t)R * line_stride * cs, (cuuint64_t)ostride * cs};
    const cuuint32_t box[4] = {(cuuint32_t)(2 * B), 1, 64, 1};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult cr = enc(tmap, sizeof(T) == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 4,
                      const_cast<void *>(src), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return cr == CUDA_SUCCESS;                                 // a shape the encoder refuses: older kernels
}

// TMA-pipelined line pass (k_fft_lines_tma) where it applies: N in {256, 512, 1024}, 16-byte aligned rows (always true
// for c16 fields; c8 fields with an odd row length -- the y pass over Nz/2+1 columns -- keep the register-I/O kernel).
// *done = false: not applicable, the caller falls back.  d_total: rows of the peer field (peer stores only).
template <typename T>
static int launch_lines_tma(const void *src, void *dst, void *const *peer_host, int P, int N, int64_t line_stride,
                            int64_t n_inner, int64_t n_outer, int64_t outer_stride, int64_t outer_start, int inverse,
                            double scale, cudaStream_t s, int64_t d_total, bool *done) {
    typedef typename C2<T>::type C;
    *done = false;
    if (N != 256 && N != 512 && N != 1024) return NBK_OK;
    const size_t cs = sizeof(C);
    if (n_outer > 1 && outer_stride == 0) return NBK_OK;
    const int64_t ostride = n_outer > 1 ? outer_stride : (int64_t)N * line_stride;
    CUtensorMap tmap;
    if (!encode_lines_tmap<T>(&tmap, src, N, line_stride, n_inner, n_outer, ostride)) return NBK_OK;
    const int R = N / 64;
    constexpr int B = 128 / (int)sizeof(C);                    // tile width: 128-byte rows
    int dtype = sizeof(T) == 4 ? NBK_F4 : NBK_F8;
    void *tw;
    int rc = get_twiddle(N, dtype, s, &tw);
    if (rc) return rc;
    // ring: R slots of the tile being transformed + P prefetch slots, sized for tma_ctas_per_sm(R) CTAs per SM
    const size_t slot = (size_t)64 * B * cs;
    const size_t fixed = (size_t)(N + 64) * cs + 26 * 8 + 64;
    const int per_sm = tma_ctas_per_sm(R);
    int NS = (int)(((size_t)(226 * 1024) / per_sm - 1024 - fixed) / slot);
    if (NS > 26) NS = 26;
    if (NS > 2 * R) NS = 2 * R;
    NBK_CHECK_ARG(NS >= R + 1, "fft_lines: the slot ring does not fit in shared memory (N = %d)", N);
    const size_t smem = (size_t)NS * slot + fixed;
    const int64_t tiles_inner = (n_inner + B - 1) / B;
    const int64_t n_tiles = tiles_inner * n_outer;
    const int64_t g = n_tiles < (int64_t)NBK_SM_COUNT * per_sm ? n_tiles : (int64_t)NBK_SM_COUNT * per_sm;
    PeerPtrs<C> peers;
    for (int i = 0; i < NBK_MAX_PEERS; i++) peers.p[i] = (peer_host && i < P) ? (C *)peer_host[i] : nullptr;
    const int n_per = peer_host ? N / P : N;
#define LAUNCH_TMA2(RR, BB, NTT, PEERF)                                                                                \
    do {                                                                                                               \
        NBK_CUDA(cudaFuncSetAttribute(k_fft_lines_tma<T, RR, BB, NTT, PEERF>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        k_fft_lines_tma<T, RR, BB, NTT, PEERF><<<(int)g, NTT, smem, s>>>(tmap, (C *)dst, peers, (const C *)tw, line_stride, n_inner, \
            tiles_inner, n_tiles, outer_stride, n_per, d_total, outer_start, inverse, (T)scale, NS);                  \
    } while (0)
#define LAUNCH_TMA(RR, BB, NTT) do { if (peer_host) LAUNCH_TMA2(RR, BB, NTT, true); else LAUNCH_TMA2(RR, BB, NTT, false); } while (0)
    if (R == 16) LAUNCH_TMA(16, B, 512);
    else if (R == 8) LAUNCH_TMA(8, B, 256);
    else LAUNCH_TMA(4, B, 128);
#undef LAUNCH_TMA
#undef LAUNCH_TMA2
    NBK_LAUNCHED();
    *done = true;
    return NBK_OK;
}

// ---------------------------------------------------------------------------------------------
// x pass fused with the FFTPower 1d auto-power binning (one rank: lines of N = 64 R strided by Ny*Nzc).  FFTPower keeps
// only the binned sums, so the transformed field is never stored: the pass reads the z + y output once, writes nothing.
// A tile runs the row-group FFTs and the radix-R combine of k_fft_lines_tma and scales each mode exactly as its store
// does.  The combine reads its R slots into registers and frees them at once: the next tile's boxes are issued before
// the radix-R DFT, so they land while this tile is transformed and binned.  Each thread then stages the power |X|^2 of
// its modes in `stage` ([B][N/2 + 2] doubles, its own area, not the ring), adding the mirror -j's power onto j's in a
// second pass (p_j + p_-j, no atomics).  A warp walks 32 consecutive j = jx >= 0 at a time along one (ky, kz) column,
// whose coordinates, compensation and weight it forms once, and whose modes it keeps from a mu division each when the
// column's smallest |k| already puts mu in [-1, 1); -j has the same |k| and mu as j for a line of sight along z.
// |k| grows with j, so equal bins are contiguous runs of lanes, which a segmented shuffle reduction folds into one
// shared-memory atomic per run; each CTA adds its sums to the global ones at the end.
// The bin of a mode must be the one nbk_power_bin gives it (binning.cu is built with --fmad=false, this file is not), so
// its arithmetic uses explicit round-to-nearest intrinsics throughout.
// The ring set-up and refill repeat k_fft_lines_tma's on purpose: the same code behind a shared helper struct measured
// 0.8 ms slower at 1024^3 f8 (8.7 against 7.9 ms per call on an H100 80GB HBM3, 700 W).
template <typename T, int R, int B, int NT>
__global__ void __launch_bounds__(NT, tma_ctas_per_sm(R))
k_fft_x_bin(const __grid_constant__ CUtensorMap tmap, const typename C2<T>::type *__restrict__ twg, int64_t n_inner,
            int64_t n_tiles, T scale, int NS, const XBinArgs a) {
    typedef typename C2<T>::type C;
    constexpr int S = 64, N = S * R, SLOT = S * B, NW = NT / 32, IT = S * B / NT;
    // staged powers: row pitch SP = 2 (mod 16) doubles, so a half warp's phase stores (8 columns x 2 consecutive j) and
    // the Nyquist reads (one column per lane) hit 16 distinct 8-byte bank pairs; the binning reads 32 consecutive j
    constexpr int SP = N / 2 + 2;
    // a warp bins IPW items of 32 j, JPW of them along one column before the next column
    constexpr int IPW = B * R / NW, JPW = IPW < R ? IPW : R;
    static_assert((S * B) % NT == 0 && B <= 32 && (B * R) % NW == 0 && IPW % JPW == 0 && R % JPW == 0, "tile geometry");
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    C *ring = reinterpret_cast<C *>(smem_raw);                 // [NS][64][B]
    C *twN = ring + (size_t)NS * SLOT;
    C *tw64 = twN + N;
    uint64_t *bars = reinterpret_cast<uint64_t *>(tw64 + S);   // [NS]
    double *stage = reinterpret_cast<double *>(bars + NS);     // [B][SP]: p_j + p_-j of column b at b * SP + j, j <= N/2
    double *s_k2 = stage + B * SP;                             // [nedge]
    const int nedge = a.nedge, nkb = nedge + 1;
    double *s_x = s_k2 + nedge;                                // per k bin (mu bin 1): sum |k| w, sum P w, sum w
    double *s_p = s_x + nkb;
    unsigned *s_n = reinterpret_cast<unsigned *>(s_p + nkb);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
        for (int i = 0; i < NS; i++) fm_mbar_init(&bars[i], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = tid; i < N; i += NT) twN[i] = twg[i];
    for (int i = tid; i < S; i += NT) tw64[i] = twg[i * R];
    for (int i = tid; i < nedge; i += NT) s_k2[i] = a.k2edges[i];
    for (int i = tid; i < nkb; i += NT) { s_x[i] = 0.0; s_p[i] = 0.0; s_n[i] = 0u; }
    __syncthreads();
    const int64_t first = blockIdx.x;
    const int my_tiles = first < n_tiles ? (int)((n_tiles - first + gridDim.x - 1) / gridDim.x) : 0;
    const int G = my_tiles * R;
    int issued = 0;
    auto issue = [&](int g) {
        const int it = g / R, j = g - it * R;
        const int64_t inner0 = (first + (int64_t)it * gridDim.x) * B;
        const int slot = g % NS;
        fm_mbar_expect_tx(&bars[slot], (unsigned)(SLOT * sizeof(C)));
        fm_tma_load_4d(ring + (size_t)slot * SLOT, &tmap, (int)(2 * inner0), j, 0, 0, &bars[slot]);
    };
    if (tid == 0) {
        const int upto = G < NS ? G : NS;
        for (; issued < upto; issued++) issue(issued);
    }
    const int Ny = a.N[1], Nz = a.N[2], Nzc = a.Nzc;
    const float kfx = a.kf32[0], kfy = a.kf32[1], kfz = a.kf32[2];
    const unsigned FULL = 0xffffffffu;
    for (int it = 0; it < my_tiles; it++) {
        const int inner0 = (int)((first + (int64_t)it * gridDim.x) * B);
        const int bvalid = (int)((n_inner - inner0) < B ? (n_inner - inner0) : B);
        const int g0 = it * R, base = g0 % NS;
        lines_tma_groups<T, R, B, NT>(ring, bars, NS, g0, tw64, (T)1);
        // ---- radix-R combine: the tile's slots -> registers, then the slots are refilled with the next tile's groups
        C v[IT][R];
#pragma unroll
        for (int i = 0; i < IT; i++) {
            const int w = tid + NT * i, b = w % B, k = w / B;
            const int pos = ((k & 7) << 3) | (k >> 3);
#pragma unroll
            for (int j = 0; j < R; j++) {
                int sj = base + j;
                if (sj >= NS) sj -= NS;
                const C x = ring[(size_t)sj * SLOT + pos * B + b];
                v[i][j] = j ? cmul(x, twN[j * k]) : x;
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic accesses to the slots before the next TMA writes
        __syncthreads();
        if (tid == 0) {
            int upto = (it + 1) * R + NS;
            if (upto > G) upto = G;
            for (; issued < upto; issued++) issue(issued);
        }
        // ---- DFT, scaled as the store of k_fft_lines_tma scales; powers of modes K = k + 64 m <= N/2 to the stage,
        // then those of K > N/2 added onto their mirror N - K
        double pw[IT][R];
#pragma unroll
        for (int i = 0; i < IT; i++) {
            const int w = tid + NT * i, b = w % B, k = w / B;
            dftR<R, C>(v[i]);
#pragma unroll
            for (int m = 0; m < R; m++) {
                const C c = C{v[i][m].x * scale, v[i][m].y * scale};
                pw[i][m] = __dadd_rn(__dmul_rn((double)c.x, (double)c.x), __dmul_rn((double)c.y, (double)c.y));
                const int K = k + S * m;
                if (K <= N / 2) stage[b * SP + K] = pw[i][m];
            }
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < IT; i++) {
            const int w = tid + NT * i, b = w % B, k = w / B;
#pragma unroll
            for (int m = R / 2; m < R; m++) {
                const int K = k + S * m;
                if (K > N / 2) stage[b * SP + N - K] = __dadd_rn(stage[b * SP + N - K], pw[i][m]);
            }
        }
        __syncthreads();
        // ---- binning.  What depends on the column b alone: its (ky, kz) coordinates, compensation and weight.
        struct Col { int iy, kz; float ky2, kz2, kzl; bool nonsing, yz0, mu_in; unsigned w; double wd, cy, cz; };
        auto column = [&](int b) {
            Col c;
            const int inner = inner0 + b;
            c.iy = inner / Nzc;
            c.kz = inner - c.iy * Nzc;
            const int jy = nbk_freq(c.iy, Ny), jz = nbk_freq(c.kz, Nz);
            const float ky = __fmul_rn((float)jy, kfy), kzv = __fmul_rn((float)jz, kfz);
            c.ky2 = __fmul_rn(ky, ky);
            c.kz2 = __fmul_rn(kzv, kzv);
            c.kzl = __fmul_rn(kzv, a.losz32);
            c.nonsing = jz > 0;                                        // Hermitian weight: 1 on the kz = 0 / Nz/2 planes
            c.w = c.nonsing ? 2u : 1u;
            c.wd = c.nonsing ? 2.0 : 1.0;
            c.yz0 = jy == 0 && jz == 0;
            // |k| of a mode is at least that of jx = 0 (each rounded step is monotone), so its |mu| = |kzl| / |k|
            // rounded is at most that of jx = 0: when mu of jx = 0 lies in [-1, 1), every mode of the column is in mu bin 1
            const float kn0 = __fsqrt_rn(__fadd_rn(__fadd_rn(0.0f, c.ky2), c.kz2));
            const float mu0 = kn0 == 0.0f ? 0.0f : __fdiv_rn(c.kzl, kn0);
            c.mu_in = kn0 != 0.0f && mu0 >= -1.0f && mu0 < 1.0f;
            c.cy = a.ct0 ? a.ct1[c.iy] : 0.0;
            c.cz = a.ct0 ? a.ctz[c.kz] : 0.0;
            return c;
        };
        // stats of mode j of column b, its power p (with the mirror's when `pair`): k bin, mu bin, weight, weighted |k|, P
        auto mode_stats = [&](const Col &c, int j, double p, bool pair, int &kb, int &dm, unsigned &cnt, double &xs,
                              double &ps) {
            const int jx = nbk_freq(j, N);
            const float kx = __fmul_rn((float)jx, kfx);
            const float k2 = __fadd_rn(__fadd_rn(__fmul_rn(kx, kx), c.ky2), c.kz2);
            const float kn = __fsqrt_rn(k2);
            kb = nbk_k2_bin(s_k2, nedge, (double)k2, (double)kn, a.kmin, a.inv_dk, a.uniform);
            dm = 1;
            if (!c.mu_in) {
                const float mu = kn == 0.0f ? 0.0f : __fdiv_rn(c.kzl, kn);
                dm = (mu >= -1.0f ? 1 : 0) + (mu >= 1.0f ? 1 : 0);   // numpy.digitize(mu, [-1, 1])
            }
            cnt = pair ? 2u * c.w : c.w;
            xs = __dmul_rn((double)kn, pair ? 2.0 * c.wd : c.wd);
            double vol = a.volume;
            if (a.ct0) vol = __dmul_rn(__dmul_rn(vol, __dmul_rn(a.ct0[j], c.cy)), c.cz);
            ps = (jx == 0 && c.yz0) ? 0.0 : __dmul_rn(p, vol);     // the zero mode is cleared
            if (c.nonsing) ps = __dmul_rn(ps, 2.0);
        };
        // modes outside mu bin 1 (mu == 1 on the kz axis, a rounding below -1) go straight to the global sums
        auto add_global = [&](int key, unsigned cnt, double xs, double ps) {
            atomicAdd(&a.nsum[key], (unsigned long long)cnt);
            if (xs != 0.0) atomicAdd(&a.xsum[key], xs);
            if (ps != 0.0) atomicAdd(&a.ysum[2 * key], ps);
        };
        for (int t0 = warp * IPW; t0 < (warp + 1) * IPW; t0 += JPW) {
            const int b = t0 / R;
            if (b >= bvalid) break;
            const Col col = column(b);
            for (int jb = t0 - b * R; jb < t0 - b * R + JPW; jb++) {
                const int j = jb * 32 + lane;                           // j < N / 2: pairs (j, N - j), j = 0 alone
                int kb, dm;
                unsigned cnt;
                double xs, ps;
                mode_stats(col, j, stage[b * SP + j], j > 0, kb, dm, cnt, xs, ps);
                int key = kb;
                if (dm != 1) { add_global(kb * 3 + dm, cnt, xs, ps); key = -1; cnt = 0; xs = 0.0; ps = 0.0; }
                // equal-key runs of lanes -> one atomic per run
                const int prev = __shfl_up_sync(FULL, key, 1);
                const bool head = (lane == 0) || (prev != key);
                const unsigned heads = __ballot_sync(FULL, head);
                if (heads == 1u) {
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) {
                        cnt += __shfl_xor_sync(FULL, cnt, o);
                        xs += __shfl_xor_sync(FULL, xs, o);
                        ps += __shfl_xor_sync(FULL, ps, o);
                    }
                } else if (heads != FULL) {
                    // step o runs while some run is longer than o, i.e. o consecutive lanes are no heads; lane + o
                    // is in this lane's run when none of lanes lane + 1 .. lane + o is a head
                    unsigned more = ~heads;                             // lanes that continue a run
                    for (int o = 1; more; o <<= 1) {
                        const bool take = (lane + o < 32) && ((heads >> lane >> 1) & ((1u << o) - 1u)) == 0u;
                        const unsigned c_o = __shfl_down_sync(FULL, cnt, o);
                        const double x_o = __shfl_down_sync(FULL, xs, o);
                        const double p_o = __shfl_down_sync(FULL, ps, o);
                        if (take) { cnt += c_o; xs += x_o; ps += p_o; }
                        more &= more >> o;                              // lanes starting o more continuing lanes
                    }
                }
                if (head && key >= 0) {
                    atomicAdd(&s_n[key], cnt);
                    if (xs != 0.0) atomicAdd(&s_x[key], xs);
                    if (ps != 0.0) atomicAdd(&s_p[key], ps);
                }
            }
        }
        // the Nyquist modes jx = -N/2 (no mirror), one lane per column
        if (warp == NW - 1 && lane < bvalid) {
            int kb, dm;
            unsigned cnt;
            double xs, ps;
            mode_stats(column(lane), N / 2, stage[lane * SP + N / 2], false, kb, dm, cnt, xs, ps);
            if (dm != 1) add_global(kb * 3 + dm, cnt, xs, ps);
            else {
                atomicAdd(&s_n[kb], cnt);
                if (xs != 0.0) atomicAdd(&s_x[kb], xs);
                if (ps != 0.0) atomicAdd(&s_p[kb], ps);
            }
        }
        // the next tile's stage stores follow the CTA barriers of its row-group FFTs and its combine
    }
    __syncthreads();
    for (int i = tid; i < nkb; i += NT) {
        const int key = i * 3 + 1;
        if (s_n[i]) atomicAdd(&a.nsum[key], (unsigned long long)s_n[i]);
        if (s_x[i] != 0.0) atomicAdd(&a.xsum[key], s_x[i]);
        if (s_p[i] != 0.0) atomicAdd(&a.ysum[2 * key], s_p[i]);
    }
}

template <typename T>
static int launch_x_bin(void *cplx, double scale, const XBinArgs &a, cudaStream_t s, bool *done) {
    typedef typename C2<T>::type C;
    *done = false;
    const int N = a.N[0];
    if (N != 256 && N != 512 && N != 1024) return NBK_OK;
    const int64_t line_stride = (int64_t)a.N[1] * a.Nzc;
    CUtensorMap tmap;
    if (!encode_lines_tmap<T>(&tmap, cplx, N, line_stride, line_stride, 1, (int64_t)N * line_stride)) return NBK_OK;
    const int R = N / 64;
    constexpr int B = 128 / (int)sizeof(C);
    const size_t cs = sizeof(C), slot = (size_t)64 * B * cs;
    // as k_fft_lines_tma's ring, less the staged powers (B (N/2 + 2) doubles: 4 slots at N = 1024) and the edges and
    // accumulators (20 B per k bin + the f8 edges: close to 2 slots at N = 1024 with its N/2 default bins).  The slots are
    // freed before the radix-R DFT, so R + 1 of them keep the next tile's boxes in flight through the DFT and binning.
    const size_t fixed = (size_t)(N + 64) * cs + 26 * 8 + (size_t)B * (N / 2 + 2) * 8 + (size_t)a.nedge * 8 +
                         (size_t)(a.nedge + 1) * 20 + 64;
    const int per_sm = tma_ctas_per_sm(R);
    const size_t budget = (size_t)(226 * 1024) / per_sm - 1024;
    if (budget < fixed + (size_t)(R + 1) * slot) return NBK_OK;     // too many bins for shared memory
    int NS = (int)((budget - fixed) / slot);
    if (NS > 26) NS = 26;
    if (NS > 2 * R) NS = 2 * R;
    const size_t smem = (size_t)NS * slot + fixed;
    int dtype = sizeof(T) == 4 ? NBK_F4 : NBK_F8;
    void *tw;
    int rc = get_twiddle(N, dtype, s, &tw);
    if (rc) return rc;
    const int64_t n_tiles = (line_stride + B - 1) / B;
    const int64_t g = n_tiles < (int64_t)NBK_SM_COUNT * per_sm ? n_tiles : (int64_t)NBK_SM_COUNT * per_sm;
#define LAUNCH_XB(RR, NTT)                                                                                             \
    do {                                                                                                               \
        NBK_CUDA(cudaFuncSetAttribute(k_fft_x_bin<T, RR, B, NTT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        k_fft_x_bin<T, RR, B, NTT><<<(int)g, NTT, smem, s>>>(tmap, (const C *)tw, line_stride, n_tiles, (T)scale, NS, a); \
    } while (0)
    if (R == 16) LAUNCH_XB(16, 512);
    else if (R == 8) LAUNCH_XB(8, 256);
    else LAUNCH_XB(4, 128);
#undef LAUNCH_XB
    NBK_LAUNCHED();
    *done = true;
    return NBK_OK;
}

// f8 only: on f4 fields the fused pass measured slower than the x pass and nbk_power_bin it replaces (the c8 x pass is
// cheaper, the binning the same), and ptxas may contract its combine into other FMAs than k_fft_lines_tma's, which
// moves f4 modes by an ulp
int fft_x_bin_launch(void *cplx, int dtype, double scale, const XBinArgs &a, cudaStream_t s, bool *done) {
    *done = false;
    if (dtype != NBK_F8) return NBK_OK;
    return launch_x_bin<double>(cplx, scale, a, s, done);
}

// register-I/O line pass (N >= 64; the TMA pass is tried first); peer_host != nullptr selects the peer-memory scatter
// store into a field of d_total rows
template <typename T>
static int launch_lines_rg(const void *src, void *dst, void *const *peer_host, int P, int N, int64_t line_stride,
                           int64_t n_inner, int64_t n_outer, int64_t outer_stride, int64_t outer_start, int inverse,
                           double scale, cudaStream_t s, int64_t d_total) {
    typedef typename C2<T>::type C;
    {
        bool done = false;
        int rct = launch_lines_tma<T>(src, dst, peer_host, P, N, line_stride, n_inner, n_outer, outer_stride, outer_start,
                                      inverse, scale, s, d_total, &done);
        if (rct || done) return rct;
    }
    int dtype = sizeof(T) == 4 ? NBK_F4 : NBK_F8;
    void *tw;
    int rc = get_twiddle(N, dtype, s, &tw);
    if (rc) return rc;
    // tile width: 128-byte runs; the peer-memory scatter uses 256-byte runs (wider NVLink writes)
    int B = (peer_host ? 256 : 128) / (int)sizeof(C);
    if (B > 16) B = 16;
    while (B > 1 && ((size_t)N * (B + 2) * sizeof(C) > 220 * 1024 || B / 2 >= n_inner)) B >>= 1;
    size_t smem = (size_t)N * (B + 2) * sizeof(C);
    NBK_CHECK_ARG(smem <= 227 * 1024, "fft_lines: N=%d does not fit in shared memory", N);
    int64_t tiles_inner = (n_inner + B - 1) / B;
    int64_t n_tiles = tiles_inner * n_outer;
    int per_sm = (int)((227 * 1024) / (smem + 1024));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 4) per_sm = 4;
    const int nthreads = (per_sm == 1 && B >= 4) ? 512 : 256;
    if (nthreads == 256 && per_sm > 2) per_sm = 2;       // 128 registers per thread
    int64_t g = n_tiles < (int64_t)NBK_SM_COUNT * per_sm ? n_tiles : (int64_t)NBK_SM_COUNT * per_sm;
    PeerPtrs<C> peers;
    for (int i = 0; i < NBK_MAX_PEERS; i++) peers.p[i] = (peer_host && i < P) ? (C *)peer_host[i] : nullptr;
    const int n_per = peer_host ? N / P : N;
    const int first_per_thread = (int)(((int64_t)(N >> 3) * B) / nthreads);
    const bool exact = ((int64_t)(N >> 3) * B) % nthreads == 0;
#define LAUNCH_RGP(BB, NTT, IT)                                                                                       \
        if (peer_host) {                                                                                           \
            NBK_CUDA(cudaFuncSetAttribute(k_fft_lines_rgp<T, BB, true, NTT, IT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            k_fft_lines_rgp<T, BB, true, NTT, IT><<<(int)g, NTT, smem, s>>>((const C *)src, (C *)dst, peers, (const C *)tw, N, \
                ilog2(N), line_stride, n_inner, tiles_inner, n_tiles, outer_stride, n_per, d_total, outer_start, inverse, (T)scale); \
        } else {                                                                                                   \
            NBK_CUDA(cudaFuncSetAttribute(k_fft_lines_rgp<T, BB, false, NTT, IT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            k_fft_lines_rgp<T, BB, false, NTT, IT><<<(int)g, NTT, smem, s>>>((const C *)src, (C *)dst, peers, (const C *)tw, N, \
                ilog2(N), line_stride, n_inner, tiles_inner, n_tiles, outer_stride, n_per, d_total, outer_start, inverse, (T)scale); \
        }
    // the common shapes: two first-stage butterflies per thread (512^3: B=8/16, 256 threads; 1024^3: B=8, 512 threads)
    if (exact && first_per_thread == 2) {
        bool done = true;
        if (nthreads == 512 && B == 8) { LAUNCH_RGP(8, 512, 2) }
        else if (nthreads == 512 && B == 16) { LAUNCH_RGP(16, 512, 2) }
        else if (nthreads == 256 && B == 8) { LAUNCH_RGP(8, 256, 2) }
        else if (nthreads == 256 && B == 16) { LAUNCH_RGP(16, 256, 2) }
        else done = false;
        if (done) { NBK_LAUNCHED(); return NBK_OK; }
    }
#undef LAUNCH_RGP
#define LAUNCH_RG(BB, NTT)                                                                                            \
    case BB:                                                                                                       \
        if (peer_host) {                                                                                           \
            NBK_CUDA(cudaFuncSetAttribute(k_fft_lines_rg<T, BB, true, NTT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            k_fft_lines_rg<T, BB, true, NTT><<<(int)g, NTT, smem, s>>>((const C *)src, (C *)dst, peers, (const C *)tw, N, \
                ilog2(N), line_stride, n_inner, tiles_inner, n_tiles, outer_stride, n_per, d_total, outer_start, inverse, (T)scale); \
        } else {                                                                                                   \
            NBK_CUDA(cudaFuncSetAttribute(k_fft_lines_rg<T, BB, false, NTT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            k_fft_lines_rg<T, BB, false, NTT><<<(int)g, NTT, smem, s>>>((const C *)src, (C *)dst, peers, (const C *)tw, N, \
                ilog2(N), line_stride, n_inner, tiles_inner, n_tiles, outer_stride, n_per, d_total, outer_start, inverse, (T)scale); \
        }                                                                                                          \
        break;
    if (nthreads == 512) {
        switch (B) {
            LAUNCH_RG(4, 512) LAUNCH_RG(8, 512) LAUNCH_RG(16, 512)
            default: nbk_set_error("fft_lines: internal tile width %d", B); return NBK_ERR_ARG;
        }
    } else {
        switch (B) {
            LAUNCH_RG(1, 256) LAUNCH_RG(2, 256) LAUNCH_RG(4, 256) LAUNCH_RG(8, 256) LAUNCH_RG(16, 256)
            default: nbk_set_error("fft_lines: internal tile width %d", B); return NBK_ERR_ARG;
        }
    }
#undef LAUNCH_RG
    NBK_LAUNCHED();
    return NBK_OK;
}

template <typename T>
static int launch_lines(const void *data, void *dst, int N, int64_t line_stride, int64_t n_inner, int64_t n_outer,
                        int64_t outer_stride, int inverse, double scale, cudaStream_t s) {
    typedef typename C2<T>::type C;
    int dtype = sizeof(T) == 4 ? NBK_F4 : NBK_F8;
    if (N == 1) {
        if (scale != 1.0 || dst != data) {
            nbk_set_error("fft_lines: N == 1 with scale / out of place is not supported");
            return NBK_ERR_UNSUPPORTED;
        }
        return NBK_OK;
    }
    if (N >= 64)
        return launch_lines_rg<T>(data, dst, nullptr, 1, N, line_stride, n_inner, n_outer, outer_stride, 0, inverse, scale, s, 0);
    void *tw;
    int rc = get_twiddle(N, dtype, s, &tw);
    if (rc) return rc;
    // two tile buffers [N][B+1] + twiddle table [N].  B * sizeof(C) = 128 bytes makes every quarter-warp shared
    // access one full padded row (bank-conflict free for any row), so keep that width as long as it fits and run
    // one 512-thread CTA per SM; narrower tiles only for very long lines.
    int B = 128 / (int)sizeof(C);
    while (B > 1 && ((size_t)N * (2 * (B + 1) + 1) * sizeof(C) > 220 * 1024 || B / 2 >= n_inner)) B >>= 1;
    size_t smem = (size_t)N * (2 * (B + 1) + 1) * sizeof(C);
    NBK_CHECK_ARG(smem <= 227 * 1024, "fft_lines: N=%d does not fit in shared memory", N);
    int64_t tiles_inner = (n_inner + B - 1) / B;
    int64_t n_tiles = tiles_inner * n_outer;
    int per_sm = (int)((227 * 1024) / (smem + 1024));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 8) per_sm = 8;
    int64_t g = n_tiles < (int64_t)NBK_SM_COUNT * per_sm ? n_tiles : (int64_t)NBK_SM_COUNT * per_sm;
    const int nthreads = (per_sm == 1 && (int64_t)N * B >= 4096) ? 512 : 256;
#define LAUNCH_LINES(BB)                                                                                          \
    case BB:                                                                                                      \
        NBK_CUDA(cudaFuncSetAttribute(k_fft_lines<T, BB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        k_fft_lines<T, BB><<<(int)g, nthreads, smem, s>>>((const C *)data, (C *)dst, (const C *)tw, N, ilog2(N), line_stride, n_inner, \
                                                     tiles_inner, n_tiles, outer_stride, inverse, (T)scale);      \
        break;
    switch (B) {
        LAUNCH_LINES(1) LAUNCH_LINES(2) LAUNCH_LINES(4) LAUNCH_LINES(8) LAUNCH_LINES(16)
        default: nbk_set_error("fft_lines: internal tile width %d", B); return NBK_ERR_ARG;
    }
#undef LAUNCH_LINES
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_fft_lines(void *cplx, int dtype, int64_t n_line, int64_t line_stride, int64_t n_inner,
                             int64_t n_outer, int64_t outer_stride, int inverse, double scale, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "fft_lines: bad dtype %d", dtype);
    NBK_CHECK_ARG(is_pow2(n_line) && n_line <= pow2_max_line(dtype),
                  "fft_lines: line length %lld is not a power of two of at most %lld points", (long long)n_line,
                  (long long)pow2_max_line(dtype));
    if (n_inner <= 0 || n_outer <= 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == NBK_F4)
        return launch_lines<float>(cplx, cplx, (int)n_line, line_stride, n_inner, n_outer, outer_stride, inverse, scale, s);
    return launch_lines<double>(cplx, cplx, (int)n_line, line_stride, n_inner, n_outer, outer_stride, inverse, scale, s);
}

// out-of-place variant (same layout for src and dst)
extern "C" int nbk_fft_lines_oop(const void *src, void *dst, int dtype, int64_t n_line, int64_t line_stride,
                                 int64_t n_inner, int64_t n_outer, int64_t outer_stride, int inverse, double scale,
                                 void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "fft_lines_oop: bad dtype %d", dtype);
    NBK_CHECK_ARG(is_pow2(n_line) && n_line >= 2 && n_line <= pow2_max_line(dtype),
                  "fft_lines_oop: line length %lld unsupported (a power of two of at most %lld points)", (long long)n_line,
                  (long long)pow2_max_line(dtype));
    if (n_inner <= 0 || n_outer <= 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == NBK_F4)
        return launch_lines<float>(src, dst, (int)n_line, line_stride, n_inner, n_outer, outer_stride, inverse, scale, s);
    return launch_lines<double>(src, dst, (int)n_line, line_stride, n_inner, n_outer, outer_stride, inverse, scale, s);
}

// line pass whose output rows go to the P blocks of peer_host, each a field of d_total rows [N/P][d_total][n_inner]
template <typename T>
static int launch_lines_scatter(const void *src, void *const *peer_host, int N, int64_t n_inner, int64_t n_outer,
                                int64_t outer_start, int P, int inverse, double scale, cudaStream_t s, int64_t d_total) {
    if (N >= 64)
        return launch_lines_rg<T>(src, nullptr, peer_host, P, N, n_inner, n_inner, n_outer, (int64_t)N * n_inner, outer_start,
                                  inverse, scale, s, d_total);
    typedef typename C2<T>::type C;
    int dtype = sizeof(T) == 4 ? NBK_F4 : NBK_F8;
    void *tw;
    int rc = get_twiddle(N, dtype, s, &tw);
    if (rc) return rc;
    int B = pick_B(N, (int)sizeof(C), n_inner);
    size_t smem = (size_t)N * (B + 2) * sizeof(C);
    NBK_CHECK_ARG(smem <= 227 * 1024, "fft_lines_scatter: N=%d does not fit in shared memory", N);
    int64_t tiles_inner = (n_inner + B - 1) / B;
    int64_t n_tiles = tiles_inner * n_outer;
    int per_sm = (int)((227 * 1024) / (smem + 1024));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 8) per_sm = 8;
    int64_t g = n_tiles < (int64_t)NBK_SM_COUNT * per_sm ? n_tiles : (int64_t)NBK_SM_COUNT * per_sm;
    PeerPtrs<C> peers;
    for (int i = 0; i < NBK_MAX_PEERS; i++) peers.p[i] = i < P ? (C *)peer_host[i] : nullptr;
#define LAUNCH_LS(BB)                                                                                                \
    case BB:                                                                                                         \
        NBK_CUDA(cudaFuncSetAttribute(k_fft_lines_scatter<T, BB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        k_fft_lines_scatter<T, BB><<<(int)g, 256, smem, s>>>((const C *)src, peers, (const C *)tw, N, ilog2(N), n_inner, \
                                                             tiles_inner, n_tiles, N / P, d_total, outer_start,      \
                                                             inverse, (T)scale);                                     \
        break;
    switch (B) {
        LAUNCH_LS(1) LAUNCH_LS(2) LAUNCH_LS(4) LAUNCH_LS(8) LAUNCH_LS(16)
        default: nbk_set_error("fft_lines_scatter: internal tile width %d", B); return NBK_ERR_ARG;
    }
#undef LAUNCH_LS
    NBK_LAUNCHED();
    return NBK_OK;
}

template <typename T>
static int launch_z(const void *in, void *out, int64_t rows, int Nz, bool forward, double scale, cudaStream_t s) {
    typedef typename C2<T>::type C;
    int dtype = sizeof(T) == 4 ? NBK_F4 : NBK_F8;
    int M = Nz / 2;
    void *twM, *twN;
    int rc = get_twiddle(M, dtype, s, &twM);
    if (rc) return rc;
    rc = get_twiddle(Nz, dtype, s, &twN);
    if (rc) return rc;
    if (forward && (M == 128 || M == 256 || M == 512) && (reinterpret_cast<uintptr_t>(in) & 15) == 0 &&
        ((size_t)Nz * sizeof(T)) % 16 == 0) {
        // warp-per-row TMA pass: 12 warps, per-warp ring of row buffers filling the SM's shared memory
        constexpr int NWZ = 12;
        const size_t rowb = (size_t)M * sizeof(C);
        const size_t twb = ((size_t)Nz + 7 * (M / 8) + 56) * sizeof(C);       // W_N | stage-1 table | stage-2 table
        int nbuf = (int)(((size_t)224 * 1024 - twb - 1024) / (NWZ * rowb));
        if (nbuf > 4) nbuf = 4;
        if (nbuf < 2) nbuf = 2;
        const size_t smem = twb + (size_t)NWZ * nbuf * rowb + (size_t)NWZ * nbuf * 8 + 128;
        NBK_CHECK_ARG(smem <= 227 * 1024, "fft z pass: Nz=%d does not fit in shared memory", Nz);
        int64_t g = (rows + NWZ - 1) / NWZ;
        if (g > NBK_SM_COUNT) g = NBK_SM_COUNT;
#define LAUNCH_ZT(LMM)                                                                                            \
        do {                                                                                                      \
            NBK_CUDA(cudaFuncSetAttribute(k_fft_z_r2c_tma<T, LMM, NWZ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            k_fft_z_r2c_tma<T, LMM, NWZ><<<(int)g, 32 * NWZ, smem, s>>>((const T *)in, (C *)out, (const C *)twN, rows, (T)scale, nbuf); \
        } while (0)
        if (M == 512) LAUNCH_ZT(9); else if (M == 256) LAUNCH_ZT(8); else LAUNCH_ZT(7);
#undef LAUNCH_ZT
        NBK_LAUNCHED();
        return NBK_OK;
    }
    if (forward && M >= 64 && M <= 256 * (sizeof(T) == 4 ? 16 : 8)) {   // the tile must fit the registers
        // register-I/O variant: 256 threads hold the whole tile across the last stage (M * B <= 256 V)
        const int V = sizeof(T) == 4 ? 16 : 8;
        int B = 16;
        while (B > 1 && (M * B > 256 * V || B / 2 >= rows)) B >>= 1;
        size_t smem = ((size_t)M * (B + 1) + Nz + 7 * (M / 8)) * sizeof(C);   // tile | W_N | first-stage twiddles
        NBK_CHECK_ARG(smem <= 227 * 1024, "fft z pass: Nz=%d does not fit in shared memory", Nz);
        int64_t n_tiles = (rows + B - 1) / B;
        int per_sm = (int)((227 * 1024) / (smem + 1024));
        if (per_sm < 1) per_sm = 1;
        if (per_sm > 4) per_sm = 4;
        int64_t g = n_tiles < (int64_t)NBK_SM_COUNT * per_sm ? n_tiles : (int64_t)NBK_SM_COUNT * per_sm;
#define LAUNCH_ZRG(BB)                                                                                            \
    case BB: {                                                                                                    \
        NBK_CUDA(cudaFuncSetAttribute(k_fft_z_r2c_rg<T, BB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        int occ = 1;   /* persistent tile loop: exactly one wave of resident CTAs (registers, not shared memory, limit it) */ \
        NBK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_fft_z_r2c_rg<T, BB>, 256, smem));           \
        if (occ < 1) occ = 1;                                                                                     \
        if (g > (int64_t)NBK_SM_COUNT * occ) g = (int64_t)NBK_SM_COUNT * occ;                                      \
        k_fft_z_r2c_rg<T, BB><<<(int)g, 256, smem, s>>>((const T *)in, (C *)out, (const C *)twN, Nz, ilog2(M), rows, (T)scale); \
        break; }
        switch (B) {
            LAUNCH_ZRG(1) LAUNCH_ZRG(2) LAUNCH_ZRG(4) LAUNCH_ZRG(8) LAUNCH_ZRG(16)
            default: nbk_set_error("fft z pass: internal tile width %d", B); return NBK_ERR_ARG;
        }
#undef LAUNCH_ZRG
        NBK_LAUNCHED();
        return NBK_OK;
    }
    int B = pick_B(M, (int)sizeof(C), rows);
    size_t smem = ((size_t)M * (B + 2) + 8) * sizeof(C);     // tile [M][B+1] (+8 skew) + twiddle table [M]
    NBK_CHECK_ARG(smem <= 227 * 1024, "fft z pass: Nz=%d does not fit in shared memory", Nz);
    int64_t n_tiles = (rows + B - 1) / B;
    int per_sm = (int)((227 * 1024) / (smem + 1024));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 8) per_sm = 8;
    int64_t g = n_tiles < (int64_t)NBK_SM_COUNT * per_sm ? n_tiles : (int64_t)NBK_SM_COUNT * per_sm;
#define LAUNCH_Z(BB)                                                                                              \
    case BB:                                                                                                      \
        if (forward) {                                                                                            \
            NBK_CUDA(cudaFuncSetAttribute(k_fft_z_r2c<T, BB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            k_fft_z_r2c<T, BB><<<(int)g, 256, smem, s>>>((const T *)in, (C *)out, (const C *)twM, (const C *)twN, Nz, \
                                                         ilog2(M), rows, (T)scale);                               \
        } else {                                                                                                  \
            NBK_CUDA(cudaFuncSetAttribute(k_fft_z_c2r<T, BB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            k_fft_z_c2r<T, BB><<<(int)g, 256, smem, s>>>((const C *)in, (T *)out, (const C *)twM, (const C *)twN, Nz, \
                                                         ilog2(M), rows);                                         \
        }                                                                                                         \
        break;
    switch (B) {
        LAUNCH_Z(1) LAUNCH_Z(2) LAUNCH_Z(4) LAUNCH_Z(8) LAUNCH_Z(16)
        default: nbk_set_error("fft z pass: internal tile width %d", B); return NBK_ERR_ARG;
    }
#undef LAUNCH_Z
    NBK_LAUNCHED();
    return NBK_OK;
}

static int check_dims(const char *who, int dtype, int64_t Nx, int64_t Ny, int64_t Nz) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "%s: bad dtype %d", who, dtype);
    const int64_t ml = pow2_max_line(dtype);
    NBK_CHECK_ARG(is_pow2(Nx) && is_pow2(Ny) && is_pow2(Nz) && Nz >= 4 && Nx <= ml && Ny <= ml && Nz <= 2 * ml,
                  "%s: Nmesh (%lld,%lld,%lld) unsupported: each side must be a power of two (Nz >= 4), Nx and Ny at "
                  "most %lld and Nz at most %lld in %s", who, (long long)Nx, (long long)Ny, (long long)Nz,
                  (long long)ml, (long long)(2 * ml), dtype == NBK_F4 ? "f4" : "f8");
    return NBK_OK;
}

// z pass alone: real rows [rows][Nz] -> complex rows [rows][Nz/2+1]
extern "C" int nbk_fft_z_forward(const void *real, void *cplx, int dtype, int64_t rows, int64_t Nz, void *stream) {
    int rc = check_dims("fft_z_forward", dtype, 1, 1, Nz);
    if (rc) return rc;
    if (rows <= 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    return (dtype == NBK_F4) ? launch_z<float>(real, cplx, rows, (int)Nz, true, 1.0, s)
                             : launch_z<double>(real, cplx, rows, (int)Nz, true, 1.0, s);
}

// Ticket counter and per-(plane, z item) epoch flags of k_fft_zy_r2c_pipe, one set per (device, stream).  Calls on one
// stream run one after the other, so they can share a set; calls on different streams may run at the same time and
// each stream has its own.  Streams are told apart by cudaStreamGetId, which no later stream reuses (a handle can be
// reused after cudaStreamDestroy while the destroyed stream's work is still running).  A set stays allocated for the
// life of the process, as the twiddle tables do: 4 bytes plus 4 per (plane, z item) of the largest call on the stream.
struct ZyPipeSync {
    unsigned *ticket = nullptr, *flags = nullptr;
    int64_t n_flags = 0;
    unsigned epoch = 0;
};
static std::mutex g_zy_mutex;
static std::map<std::pair<int, unsigned long long>, ZyPipeSync> g_zy;

// the pipelined z + y pass where both passes would run their TMA kernels: f8, Nz = 2M with M in {128, 256, 512},
// Ny = 64 R with R in {4, 8, 16}, and more than D planes.  *done = false: not applicable, the caller runs the two passes.
template <typename T>
static int launch_zy_pipe(const void *real, void *cplx, int64_t x_n, int Ny, int Nz, cudaStream_t s, bool *done) {
    typedef typename C2<T>::type C;
    *done = false;
    const int M = Nz / 2, R = Ny / 64;
    if ((M != 128 && M != 256 && M != 512) || (R != 4 && R != 8 && R != 16) || x_n >= (1 << 20)) return NBK_OK;
    if ((reinterpret_cast<uintptr_t>(real) & 15) || ((size_t)Nz * sizeof(T)) % 16) return NBK_OK;
    const int64_t Nzc = M + 1;
    CUtensorMap tmap;
    if (!encode_lines_tmap<T>(&tmap, cplx, Ny, Nzc, Nzc, x_n, Ny * Nzc)) return NBK_OK;
    const int dtype = sizeof(T) == 4 ? NBK_F4 : NBK_F8;
    void *twz, *twy;
    int rc = get_twiddle(Nz, dtype, s, &twz);
    if (rc) return rc;
    rc = get_twiddle(Ny, dtype, s, &twy);
    if (rc) return rc;
    int dev = 0, sms = 0, l2 = 0;
    NBK_CUDA(cudaGetDevice(&dev));
    NBK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    NBK_CUDA(cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, dev));
    // pipeline depth: the y tiles trail the z items by D planes; the D planes waiting for their y tiles and the one
    // being transformed take at most about half the L2
    const int64_t plane_bytes = (int64_t)Ny * Nzc * (int64_t)sizeof(C);
    int64_t D = (int64_t)l2 / (2 * plane_bytes) - 1;
    if (D < 1) D = 1;
    // a slab of at most D planes fits in half the L2 as a whole: the y pass of the two launches already reads the z
    // rows from L2, and the single persistent kernel only adds its start-up (measured slower on 1- and 2-plane slabs)
    if (x_n <= D) return NBK_OK;
    // shared memory: the larger of the z row buffers and the y ring, the twiddle tables, the mbarriers, the ticket
    constexpr int NW = ZY_NT / 32, B = 128 / (int)sizeof(C);
    const int nbuf = ZY_ZBUF / M, NS = R;
    const size_t zbytes = (size_t)NW * ZY_ZBUF * sizeof(C), ybytes = (size_t)NS * 64 * B * sizeof(C);
    const size_t smem = (zbytes > ybytes ? zbytes : ybytes) + ((size_t)(2 * M + 7 * (M / 8) + 56) + Ny + 64) * sizeof(C) +
                        (size_t)(NW * nbuf + NS) * 8 + 16;
    NBK_CHECK_ARG(smem <= (size_t)227 * 1024, "fft_zy_forward: the pipelined pass does not fit in shared memory "
                  "(Ny = %d, Nz = %d)", Ny, Nz);
    const int nzi = Ny / (NW * ZY_ZPW), nyi = (int)((Nzc + B - 1) / B);
    const int64_t n_items = (int64_t)(nzi + nyi) * (x_n + D);
    unsigned *ticket, *flags, epoch;
    {
        unsigned long long sid = 0;
        NBK_CUDA(cudaStreamGetId(s, &sid));
        std::lock_guard<std::mutex> lock(g_zy_mutex);
        ZyPipeSync &st = g_zy[std::make_pair(dev, sid)];
        if (!st.ticket) {
            NBK_CUDA(cudaMalloc(&st.ticket, sizeof(unsigned)));
            NBK_CUDA(cudaMemsetAsync(st.ticket, 0, sizeof(unsigned), s));
        }
        if (st.n_flags < x_n * nzi) {
            if (st.flags) NBK_CUDA(cudaFree(st.flags));
            st.flags = nullptr;
            st.n_flags = 0;
            NBK_CUDA(cudaMalloc(&st.flags, (size_t)x_n * nzi * sizeof(unsigned)));
            NBK_CUDA(cudaMemsetAsync(st.flags, 0, (size_t)x_n * nzi * sizeof(unsigned), s));
            st.n_flags = x_n * nzi;
        }
        ticket = st.ticket;
        flags = st.flags;
        epoch = ++st.epoch;
    }
#define LAUNCH_ZY(LMM, RR)                                                                                           \
    do {                                                                                                             \
        auto kern = k_fft_zy_r2c_pipe<T, LMM, RR>;                                                                   \
        NBK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));                \
        int occ = 0;                                                                                                 \
        NBK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, ZY_NT, smem));                            \
        NBK_CHECK_ARG(occ >= 1, "fft_zy_forward: the pipelined pass cannot be resident (Ny = %d, Nz = %d)", Ny, Nz); \
        int64_t g = (int64_t)occ * sms;                                                                              \
        if (g > n_items) g = n_items;                                                                                \
        kern<<<(int)g, ZY_NT, smem, s>>>(tmap, (const T *)real, (C *)cplx, (const C *)twz, (const C *)twy, (int)x_n,  \
                                         (int)D, ticket, flags, epoch, (T)1, (T)1);                                  \
    } while (0)
#define LAUNCH_ZY_R(LMM) do { if (R == 16) LAUNCH_ZY(LMM, 16); else if (R == 8) LAUNCH_ZY(LMM, 8); else LAUNCH_ZY(LMM, 4); } while (0)
    if (M == 512) LAUNCH_ZY_R(9); else if (M == 256) LAUNCH_ZY_R(8); else LAUNCH_ZY_R(7);
#undef LAUNCH_ZY_R
#undef LAUNCH_ZY
    NBK_LAUNCHED();
    *done = true;
    return NBK_OK;
}

// z and y passes of the forward transform of x_n planes: the pipelined kernel where it applies, else the z pass and
// then the y lines
extern "C" int nbk_fft_zy_forward(const void *real, void *cplx, int dtype, int64_t x_n, int64_t Ny, int64_t Nz,
                                  void *stream) {
    int rc = check_dims("fft_zy_forward", dtype, 1, Ny, Nz);
    if (rc) return rc;
    if (x_n <= 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    int64_t Nzc = Nz / 2 + 1;
    if (dtype == NBK_F8) {
        bool done = false;
        rc = launch_zy_pipe<double>(real, cplx, x_n, (int)Ny, (int)Nz, s, &done);
        if (rc || done) return rc;
    }
    rc = (dtype == NBK_F4) ? launch_z<float>(real, cplx, x_n * Ny, (int)Nz, true, 1.0, s)
                           : launch_z<double>(real, cplx, x_n * Ny, (int)Nz, true, 1.0, s);
    if (rc) return rc;
    return nbk_fft_lines(cplx, dtype, Ny, Nzc, Nzc, x_n, Ny * Nzc, 0, 1.0, stream);
}

extern "C" int nbk_fft_zy_backward(void *cplx, void *real, int dtype, int64_t x_n, int64_t Ny, int64_t Nz,
                                   void *stream) {
    int rc = check_dims("fft_zy_backward", dtype, 1, Ny, Nz);
    if (rc) return rc;
    if (x_n <= 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    int64_t Nzc = Nz / 2 + 1;
    rc = nbk_fft_lines(cplx, dtype, Ny, Nzc, Nzc, x_n, Ny * Nzc, 1, 1.0, stream);
    if (rc) return rc;
    return (dtype == NBK_F4) ? launch_z<float>(cplx, real, x_n * Ny, (int)Nz, false, 1.0, s)
                             : launch_z<double>(cplx, real, x_n * Ny, (int)Nz, false, 1.0, s);
}

extern "C" int nbk_r2c(const void *real, void *cplx, int dtype, const int64_t *nmesh, double extra_scale, void *stream) {
    int rc = check_dims("r2c", dtype, nmesh[0], nmesh[1], nmesh[2]);
    if (rc) return rc;
    int64_t Nx = nmesh[0], Ny = nmesh[1], Nz = nmesh[2], Nzc = Nz / 2 + 1;
    rc = nbk_fft_zy_forward(real, cplx, dtype, Nx, Ny, Nz, stream);
    if (rc) return rc;
    double scale = extra_scale / ((double)Nx * (double)Ny * (double)Nz);
    if (Nx == 1) return nbk_scale(cplx, dtype, 2 * Ny * Nzc, scale, stream);
    return nbk_fft_lines(cplx, dtype, Nx, Ny * Nzc, Ny * Nzc, 1, 0, 0, scale, stream);
}

// c2r destroys its complex input unless `work` (same size as cplx) is given
extern "C" int nbk_c2r(const void *cplx, void *real, int dtype, const int64_t *nmesh, void *work, void *stream) {
    int rc = check_dims("c2r", dtype, nmesh[0], nmesh[1], nmesh[2]);
    if (rc) return rc;
    int64_t Nx = nmesh[0], Ny = nmesh[1], Nz = nmesh[2], Nzc = Nz / 2 + 1;
    void *c = const_cast<void *>(cplx);
    if (work && work != cplx) {
        size_t bytes = (size_t)Nx * Ny * Nzc * (dtype == NBK_F4 ? 8 : 16);
        NBK_CUDA(cudaMemcpyAsync(work, cplx, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
        c = work;
    }
    rc = nbk_fft_lines(c, dtype, Nx, Ny * Nzc, Ny * Nzc, 1, 0, 1, 1.0, stream);
    if (rc) return rc;
    return nbk_fft_zy_backward(c, real, dtype, Nx, Ny, Nz, stream);
}

// ---------------------------------------------------------------------------------------------
// slab <-> pencil transposes for P > 1 (row copies of Nzc complex, coalesced along kz)
// ---------------------------------------------------------------------------------------------
// generic: dst[(a*nb + b)*row + k] = src[(b*na + a)*row + k] with an extra block split described by the callers
template <typename C>
__global__ void __launch_bounds__(256)
k_row_permute(const C *__restrict__ src, C *__restrict__ dst, int64_t n_rows, int row, int64_t d0, int64_t d1,
              int64_t d2, int64_t s0, int64_t s1, int64_t s2) {
    // destination row index r = (i0*d1 + i1)*d2 + i2  ->  source row = i0*s0 + i1*s1 + i2*s2
    int lanes_per_row = 32;
    int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / lanes_per_row;
    int lane = threadIdx.x % lanes_per_row;
    int64_t nw = ((int64_t)gridDim.x * blockDim.x) / lanes_per_row;
    for (int64_t r = wid; r < n_rows; r += nw) {
        int64_t i2 = r % d2;
        int64_t i1 = (r / d2) % d1;
        int64_t i0 = r / (d2 * d1);
        const C *sp = src + (i0 * s0 + i1 * s1 + i2 * s2) * row;
        C *dp = dst + r * row;
        for (int k = lane; k < row; k += lanes_per_row) dp[k] = sp[k];
    }
}

template <typename C>
static int launch_permute(const void *src, void *dst, int64_t d0, int64_t d1, int64_t d2, int64_t s0, int64_t s1,
                          int64_t s2, int row, cudaStream_t s) {
    int64_t n_rows = d0 * d1 * d2;
    if (n_rows == 0) return NBK_OK;
    int g = nbk_grid_for(n_rows * 32, 256, 8);
    k_row_permute<C><<<g, 256, 0, s>>>((const C *)src, (C *)dst, n_rows, row, d0, d1, d2, s0, s1, s2);
    NBK_LAUNCHED();
    return NBK_OK;
}

#define PERMUTE(dtype, ...)                                                          \
    ((dtype) == NBK_F4 ? launch_permute<float2>(__VA_ARGS__) : launch_permute<double2>(__VA_ARGS__))

// [x_n][Ny][Nzc] -> [P][y_n][x_n][Nzc]   (dst rows (p, yl, x) <- src row (x, p*y_n + yl))
extern "C" int nbk_transpose_pack(const void *src, void *dst, int dtype, int64_t x_n, int64_t Ny, int64_t Nzc,
                                  int64_t P, void *stream) {
    NBK_CHECK_ARG(P > 0 && Ny % P == 0, "transpose_pack: Ny %% P != 0");
    int64_t y_n = Ny / P;
    // dst index (i0=p, i1=yl, i2=x): src row = x*Ny + p*y_n + yl
    return PERMUTE(dtype, src, dst, P, y_n, x_n, y_n, 1, Ny, (int)Nzc, (cudaStream_t)stream);
}
// [P][y_n][x_n][Nzc] (block q came from rank q) -> [y_n][Nx][Nzc], Nx = P*x_n
extern "C" int nbk_transpose_unpack(const void *src, void *dst, int dtype, int64_t y_n, int64_t Nx, int64_t Nzc,
                                    int64_t P, void *stream) {
    NBK_CHECK_ARG(P > 0 && Nx % P == 0, "transpose_unpack: Nx %% P != 0");
    int64_t x_n = Nx / P;
    // dst (i0=yl, i1=q, i2=xl): src row = (q*y_n + yl)*x_n + xl
    return PERMUTE(dtype, src, dst, y_n, P, x_n, x_n, y_n * x_n, 1, (int)Nzc, (cudaStream_t)stream);
}
// inverse of unpack: [y_n][Nx][Nzc] -> [P][y_n][x_n][Nzc]
extern "C" int nbk_transpose_pack_back(const void *src, void *dst, int dtype, int64_t y_n, int64_t Nx, int64_t Nzc,
                                       int64_t P, void *stream) {
    NBK_CHECK_ARG(P > 0 && Nx % P == 0, "transpose_pack_back: Nx %% P != 0");
    int64_t x_n = Nx / P;
    // dst (i0=q, i1=yl, i2=xl): src row = yl*Nx + q*x_n + xl
    return PERMUTE(dtype, src, dst, P, y_n, x_n, x_n, Nx, 1, (int)Nzc, (cudaStream_t)stream);
}
// inverse of pack: [P][y_n][x_n][Nzc] -> [x_n][Ny][Nzc]
extern "C" int nbk_transpose_unpack_back(const void *src, void *dst, int dtype, int64_t x_n, int64_t Ny, int64_t Nzc,
                                         int64_t P, void *stream) {
    NBK_CHECK_ARG(P > 0 && Ny % P == 0, "transpose_unpack_back: Ny %% P != 0");
    int64_t y_n = Ny / P;
    // dst (i0=x, i1=p, i2=yl): src row = (p*y_n + yl)*x_n + x
    return PERMUTE(dtype, src, dst, x_n, P, y_n, 1, y_n * x_n, x_n, (int)Nzc, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------
// Complex-dtype meshes (ParticleMesh(dtype='c16'/'c8'): pmesh then runs c2c transforms and keeps all N^3 modes,
// `ComplexField.compressed == False`, fftpower.py:572; convpower/catalog.py:151-176).  On this path the
// configuration-space field is real-valued, so its full spectrum is the Hermitian completion of the r2c result:
//   full[ix][iy][iz] = comp[ix][iy][iz]                                   iz <= Nz/2
//                    = conj(comp[(-ix) % Nx][(-iy) % Ny][Nz - iz])        iz >  Nz/2
// One read of the compressed field, one write of the full one (a c2c transform would move three times as much).
// ---------------------------------------------------------------------------------------------
template <typename C>
__global__ void __launch_bounds__(256)
k_hermitian_expand(const C *__restrict__ comp, C *__restrict__ full, int Nx, int Ny, int Nz) {
    const int Nzc = Nz / 2 + 1;
    const int64_t rows = (int64_t)Nx * Ny;
    const int lane = threadIdx.x & 31;
    const int64_t w0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = w0; row < rows; row += nw) {
        const int ix = (int)(row / Ny), iy = (int)(row - (int64_t)ix * Ny);
        const int mx = ix ? Nx - ix : 0, my = iy ? Ny - iy : 0;
        const C *a = comp + row * Nzc;
        const C *b = comp + ((int64_t)mx * Ny + my) * Nzc;
        C *o = full + row * Nz;
        for (int iz = lane; iz < Nz; iz += 32) {
            C v;
            if (iz < Nzc) v = a[iz];
            else { v = b[Nz - iz]; v.y = -v.y; }
            o[iz] = v;
        }
    }
}

template <typename C>
__global__ void __launch_bounds__(256)
k_hermitian_compress(const C *__restrict__ full, C *__restrict__ comp, int64_t rows, int Nz) {
    const int Nzc = Nz / 2 + 1;
    const int lane = threadIdx.x & 31;
    const int64_t w0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = w0; row < rows; row += nw)
        for (int iz = lane; iz < Nzc; iz += 32) comp[row * Nzc + iz] = full[row * Nz + iz];
}

extern "C" int nbk_hermitian_expand(const void *comp, void *full, int dtype, const int64_t *nmesh, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "hermitian_expand: bad dtype %d", dtype);
    NBK_CHECK_ARG(nmesh[0] >= 2 && nmesh[1] >= 2 && nmesh[2] >= 2 && nmesh[0] < (1 << 24) && nmesh[1] < (1 << 24) &&
                  nmesh[2] < (1 << 24), "hermitian_expand: Nmesh (%lld,%lld,%lld) unsupported: sides must be >= 2",
                  (long long)nmesh[0], (long long)nmesh[1], (long long)nmesh[2]);
    NBK_CHECK_ARG(comp != nullptr && full != nullptr && comp != full, "hermitian_expand: needs two distinct buffers");
    int64_t rows = nmesh[0] * nmesh[1];
    int g = nbk_grid_for(rows * 32, 256, 8);
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == NBK_F4) k_hermitian_expand<float2><<<g, 256, 0, s>>>((const float2 *)comp, (float2 *)full, (int)nmesh[0], (int)nmesh[1], (int)nmesh[2]);
    else k_hermitian_expand<double2><<<g, 256, 0, s>>>((const double2 *)comp, (double2 *)full, (int)nmesh[0], (int)nmesh[1], (int)nmesh[2]);
    NBK_LAUNCHED();
    return NBK_OK;
}

// the stored half of a full spectrum (the inverse of nbk_hermitian_expand for Hermitian fields; rows = Nx * Ny of this rank)
extern "C" int nbk_hermitian_compress(const void *full, void *comp, int dtype, int64_t rows, int64_t Nz, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "hermitian_compress: bad dtype %d", dtype);
    NBK_CHECK_ARG(rows >= 0 && Nz >= 2 && comp != full, "hermitian_compress: bad arguments");
    if (rows == 0) return NBK_OK;
    int g = nbk_grid_for(rows * 32, 256, 8);
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == NBK_F4) k_hermitian_compress<float2><<<g, 256, 0, s>>>((const float2 *)full, (float2 *)comp, rows, (int)Nz);
    else k_hermitian_compress<double2><<<g, 256, 0, s>>>((const double2 *)full, (double2 *)comp, rows, (int)Nz);
    NBK_LAUNCHED();
    return NBK_OK;
}

// ---------------------------------------------------------------------------------------------
// Fourier-space resampling to another mesh size (pmesh `Field.resample`, called from base/mesh.py:317-327 when
// compute(Nmesh=...) asks for a size other than the source's): the modes both meshes represent are copied, the rest
// of the destination is zero (down-sampling = truncation, up-sampling = zero padding; the normalised transform keeps
// amplitudes, so the mean is preserved).  Per axis a destination index maps to the source index with the same integer
// frequency label j = nbk_freq(i, N) when -m <= 2j < m, m = min(N_src, N_dst): labels [-m/2, m/2) for even m (Nyquist
// negative, meshtools.py:150-153), [-(m-1)/2, (m-1)/2] for odd m; along the Hermitian-compressed axis indices
// 0 .. m/2 map to themselves.  Single GPU, compressed layout [Nx][Ny][Nz/2+1]; any sides.
// ---------------------------------------------------------------------------------------------
template <typename C>
__global__ void __launch_bounds__(256)
k_resample_complex(const C *__restrict__ src, C *__restrict__ dst, int sx, int sy, int sz, int dx, int dy, int dz) {
    const int szc = sz / 2 + 1, dzc = dz / 2 + 1;
    const int mzc = (sz < dz ? sz : dz) / 2 + 1;
    const int64_t rows = (int64_t)dx * dy;
    const int lane = threadIdx.x & 31;
    const int64_t w0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = w0; row < rows; row += nw) {
        const int ix = (int)(row / dy), iy = (int)(row - (int64_t)ix * dy);
        const int jx = nbk_freq(ix, dx), jy = nbk_freq(iy, dy);
        const int mx = sx < dx ? sx : dx, my = sy < dy ? sy : dy;
        const bool ok = 2 * jx >= -mx && 2 * jx < mx && 2 * jy >= -my && 2 * jy < my;
        const C *s = src + ((int64_t)(jx < 0 ? jx + sx : jx) * sy + (jy < 0 ? jy + sy : jy)) * szc;
        C *d = dst + row * dzc;
        for (int iz = lane; iz < dzc; iz += 32) d[iz] = (ok && iz < mzc) ? s[iz] : C{0, 0};
    }
}

extern "C" int nbk_resample_complex(const void *src, void *dst, int dtype, const int64_t *nmesh_src,
                                    const int64_t *nmesh_dst, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "resample_complex: bad dtype %d", dtype);
    NBK_CHECK_ARG(src != nullptr && dst != nullptr && src != dst, "resample_complex: needs two distinct buffers");
    for (int d = 0; d < 3; d++)
        NBK_CHECK_ARG(nmesh_src[d] >= 2 && nmesh_dst[d] >= 2 && nmesh_src[d] < (1 << 24) && nmesh_dst[d] < (1 << 24),
                      "resample_complex: mesh sides must be in 2 .. 2^24 - 1");
    int64_t rows = nmesh_dst[0] * nmesh_dst[1];
    int g = nbk_grid_for(rows * 32, 256, 8);
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == NBK_F4)
        k_resample_complex<float2><<<g, 256, 0, s>>>((const float2 *)src, (float2 *)dst, (int)nmesh_src[0], (int)nmesh_src[1],
                                                     (int)nmesh_src[2], (int)nmesh_dst[0], (int)nmesh_dst[1], (int)nmesh_dst[2]);
    else
        k_resample_complex<double2><<<g, 256, 0, s>>>((const double2 *)src, (double2 *)dst, (int)nmesh_src[0], (int)nmesh_src[1],
                                                      (int)nmesh_src[2], (int)nmesh_dst[0], (int)nmesh_dst[1], (int)nmesh_dst[2]);
    NBK_LAUNCHED();
    return NBK_OK;
}

// ---------------------------------------------------------------------------------------------
// The same resampling on P > 1, where each rank holds the transposed y slab [y_n][Nx][Nzc].  The x and z remaps are
// local; a destination y row comes from the rank owning the source row with the same label, or from no rank.  The host
// plans which rows travel (at most two contiguous ranges per (source, destination) pair, the labels wrap) and passes
// them as up to NBK_RESAMPLE_MAX_RANGES (local first row, count) pairs in send / receive order.
//   pack   : send[k] = src row of the k-th listed row, remapped in x and z to [Nx_dst][Nzc_dst]
//   unpack : dst local row of the k-th listed row = recv[k]; rows no range lists are zero
// ---------------------------------------------------------------------------------------------
#define NBK_RESAMPLE_MAX_RANGES (2 * NBK_MAX_PEERS)
struct ResampleRanges {
    int n;
    int first[NBK_RESAMPLE_MAX_RANGES];
    int count[NBK_RESAMPLE_MAX_RANGES];
};

// (send slot k) -> local source row: the ranges laid end to end
__device__ __forceinline__ int resample_slot_row(const ResampleRanges &r, int k) {
    for (int i = 0; i < r.n; i++) {
        if (k < r.count[i]) return r.first[i] + k;
        k -= r.count[i];
    }
    return -1;
}

// local destination row -> receive slot, or -1 when no rank sends it
__device__ __forceinline__ int resample_row_slot(const ResampleRanges &r, int row) {
    int off = 0;
    for (int i = 0; i < r.n; i++) {
        if (row >= r.first[i] && row < r.first[i] + r.count[i]) return off + row - r.first[i];
        off += r.count[i];
    }
    return -1;
}

template <typename C>
__global__ void __launch_bounds__(256)
k_resample_pack(const C *__restrict__ src, C *__restrict__ send, const ResampleRanges rr, int64_t n_slots, int sx, int sz,
                int dx, int dz) {
    const int szc = sz / 2 + 1, dzc = dz / 2 + 1;
    const int mx = sx < dx ? sx : dx;
    const int mzc = (sz < dz ? sz : dz) / 2 + 1;
    const int64_t rows = n_slots * dx;
    const int lane = threadIdx.x & 31;
    const int64_t w0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = w0; row < rows; row += nw) {
        const int k = (int)(row / dx), ix = (int)(row - (int64_t)k * dx);
        const int jx = nbk_freq(ix, dx);
        const bool ok = 2 * jx >= -mx && 2 * jx < mx;
        const C *s = src + ((int64_t)resample_slot_row(rr, k) * sx + (jx < 0 ? jx + sx : jx)) * szc;
        C *d = send + row * dzc;
        for (int iz = lane; iz < dzc; iz += 32) d[iz] = (ok && iz < mzc) ? s[iz] : C{0, 0};
    }
}

template <typename C>
__global__ void __launch_bounds__(256)
k_resample_unpack(const C *__restrict__ recv, C *__restrict__ dst, const ResampleRanges rr, int64_t dst_rows, int64_t row_len) {
    const int64_t n = dst_rows * row_len;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t y = e / row_len;
        const int k = resample_row_slot(rr, (int)y);
        dst[e] = k >= 0 ? recv[(int64_t)k * row_len + (e - y * row_len)] : C{0, 0};
    }
}

// checks the (first, count) pairs against [0, n_rows) and copies them into `rr`; `total` receives the listed rows
static int resample_ranges(const char *what, const int64_t *ranges, int n_ranges, int64_t n_rows, ResampleRanges &rr,
                           int64_t &total) {
    NBK_CHECK_ARG(n_ranges >= 0 && n_ranges <= NBK_RESAMPLE_MAX_RANGES, "%s: %d row ranges, at most %d", what, n_ranges,
                  NBK_RESAMPLE_MAX_RANGES);
    NBK_CHECK_ARG(n_ranges == 0 || ranges != nullptr, "%s: ranges missing", what);
    rr.n = n_ranges;
    total = 0;
    for (int i = 0; i < n_ranges; i++) {
        const int64_t a = ranges[2 * i], c = ranges[2 * i + 1];
        NBK_CHECK_ARG(a >= 0 && c >= 0 && a + c <= n_rows, "%s: row range %d (%lld, %lld) outside the %lld local rows", what,
                      i, (long long)a, (long long)c, (long long)n_rows);
        rr.first[i] = (int)a;
        rr.count[i] = (int)c;
        total += c;
    }
    return NBK_OK;
}

static int resample_sides(const char *what, const int64_t *nmesh_src, const int64_t *nmesh_dst) {
    NBK_CHECK_ARG(nmesh_src != nullptr && nmesh_dst != nullptr, "%s: Nmesh missing", what);
    for (int d = 0; d < 3; d++)
        NBK_CHECK_ARG(nmesh_src[d] >= 2 && nmesh_dst[d] >= 2 && nmesh_src[d] < (1 << 24) && nmesh_dst[d] < (1 << 24),
                      "%s: mesh sides must be in 2 .. 2^24 - 1", what);
    return NBK_OK;
}

extern "C" int nbk_resample_pack(const void *src, void *send, int dtype, const int64_t *nmesh_src, const int64_t *nmesh_dst,
                                 int64_t src_rows, const int64_t *ranges, int n_ranges, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "resample_pack: bad dtype %d", dtype);
    if (resample_sides("resample_pack", nmesh_src, nmesh_dst) != NBK_OK) return NBK_ERR_ARG;
    NBK_CHECK_ARG(src_rows >= 0 && src_rows <= nmesh_src[1], "resample_pack: %lld local rows of a side %lld",
                  (long long)src_rows, (long long)nmesh_src[1]);
    ResampleRanges rr;
    int64_t slots;
    if (resample_ranges("resample_pack", ranges, n_ranges, src_rows, rr, slots) != NBK_OK) return NBK_ERR_ARG;
    if (slots == 0) return NBK_OK;
    NBK_CHECK_ARG(src != nullptr && send != nullptr && src != send, "resample_pack: needs two distinct buffers");
    int g = nbk_grid_for(slots * nmesh_dst[0] * 32, 256, 8);
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == NBK_F4)
        k_resample_pack<float2><<<g, 256, 0, s>>>((const float2 *)src, (float2 *)send, rr, slots, (int)nmesh_src[0],
                                                  (int)nmesh_src[2], (int)nmesh_dst[0], (int)nmesh_dst[2]);
    else
        k_resample_pack<double2><<<g, 256, 0, s>>>((const double2 *)src, (double2 *)send, rr, slots, (int)nmesh_src[0],
                                                   (int)nmesh_src[2], (int)nmesh_dst[0], (int)nmesh_dst[2]);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_resample_unpack(const void *recv, void *dst, int dtype, const int64_t *nmesh_dst, int64_t dst_rows,
                                   const int64_t *ranges, int n_ranges, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "resample_unpack: bad dtype %d", dtype);
    if (resample_sides("resample_unpack", nmesh_dst, nmesh_dst) != NBK_OK) return NBK_ERR_ARG;
    NBK_CHECK_ARG(dst_rows >= 0 && dst_rows <= nmesh_dst[1], "resample_unpack: %lld local rows of a side %lld",
                  (long long)dst_rows, (long long)nmesh_dst[1]);
    ResampleRanges rr;
    int64_t slots;
    if (resample_ranges("resample_unpack", ranges, n_ranges, dst_rows, rr, slots) != NBK_OK) return NBK_ERR_ARG;
    for (int i = 0; i < n_ranges; i++)
        for (int j = 0; j < i; j++)
            NBK_CHECK_ARG(rr.first[i] + rr.count[i] <= rr.first[j] || rr.first[j] + rr.count[j] <= rr.first[i],
                          "resample_unpack: row ranges %d and %d overlap", j, i);
    if (dst_rows == 0) return NBK_OK;
    NBK_CHECK_ARG(dst != nullptr && (slots == 0 || (recv != nullptr && recv != dst)),
                  "resample_unpack: needs two distinct buffers");
    const int64_t row_len = nmesh_dst[0] * (nmesh_dst[2] / 2 + 1);
    int g = nbk_grid_for(dst_rows * row_len, 256, 8);
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == NBK_F4) k_resample_unpack<float2><<<g, 256, 0, s>>>((const float2 *)recv, (float2 *)dst, rr, dst_rows, row_len);
    else k_resample_unpack<double2><<<g, 256, 0, s>>>((const double2 *)recv, (double2 *)dst, rr, dst_rows, row_len);
    NBK_LAUNCHED();
    return NBK_OK;
}

// ---------------------------------------------------------------------------------------------
// Slab transpose as "line pass into send blocks" + bulk peer copies (P > 1).  The line pass (y pass of r2c, inverse x
// pass of c2r) stores its output rows directly in transposed order into P contiguous LOCAL blocks
//     send[p][kl][outer][inner]      kl = k % (N/P) the line frequency inside rank p's share, outer < n_outer
// and nbk_slab_push_range() moves block p into rank p's field [N/P][n_outer * P][n_inner] with one strided bulk copy per
// peer: rows of n_outer * n_inner contiguous elements (1 MB at 1024^3 on 8 GPUs) travel over NVLink on the copy
// engines at link rate, instead of 128..256-byte remote stores from the line pass.
// Both work on the outer sub-range [o0, o0 + o_cnt) of the slab (the send blocks keep their full [kl][n_outer][inner]
// shape): the caller pushes one part of the slab while the next part is still being transformed.
// ---------------------------------------------------------------------------------------------
extern "C" int nbk_fft_lines_pack_range(const void *src, void *send, int dtype, int64_t n_line, int64_t n_inner,
                                        int64_t n_outer, int64_t o0, int64_t o_cnt, int P, int inverse, double scale,
                                        void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "fft_lines_pack_range: bad dtype %d", dtype);
    NBK_CHECK_ARG(is_pow2(n_line) && n_line >= 2 && n_line <= pow2_max_line(dtype),
                  "fft_lines_pack_range: line length %lld unsupported (a power of two of at most %lld points)",
                  (long long)n_line, (long long)pow2_max_line(dtype));
    NBK_CHECK_ARG(P >= 1 && P <= NBK_MAX_PEERS && n_line % P == 0, "fft_lines_pack_range: bad peer count %d", P);
    NBK_CHECK_ARG(o0 >= 0 && o_cnt >= 0 && o0 + o_cnt <= n_outer, "fft_lines_pack_range: bad sub-range");
    if (n_inner <= 0 || o_cnt <= 0) return NBK_OK;
    const size_t cs = dtype == NBK_F4 ? 8 : 16;
    const size_t block = (size_t)(n_line / P) * n_outer * n_inner * cs;
    void *blocks[NBK_MAX_PEERS];
    for (int p = 0; p < P; p++) blocks[p] = (char *)send + (size_t)p * block;
    const char *sub = (const char *)src + (size_t)o0 * n_line * n_inner * cs;
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == NBK_F4)
        return launch_lines_scatter<float>(sub, blocks, (int)n_line, n_inner, o_cnt, o0, P, inverse, scale, s, n_outer);
    return launch_lines_scatter<double>(sub, blocks, (int)n_line, n_inner, o_cnt, o0, P, inverse, scale, s, n_outer);
}

extern "C" int nbk_slab_push_range(const void *send, void *const *peer_ptrs_host, int dtype, int64_t rows_per_peer,
                                   int64_t n_outer, int64_t n_inner, int64_t outer_start, int64_t o0, int64_t o_cnt, int P,
                                   int rank, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "slab_push_range: bad dtype %d", dtype);
    NBK_CHECK_ARG(P >= 1 && P <= NBK_MAX_PEERS && rank >= 0 && rank < P, "slab_push_range: bad peer count / rank");
    NBK_CHECK_ARG(o0 >= 0 && o_cnt >= 0 && o0 + o_cnt <= n_outer, "slab_push_range: bad sub-range");
    if (rows_per_peer <= 0 || o_cnt <= 0 || n_inner <= 0) return NBK_OK;
    const size_t cs = dtype == NBK_F4 ? 8 : 16;
    const size_t spitch = (size_t)n_outer * n_inner * cs;           // one kl row of my block
    const size_t dpitch = spitch * P;                               // the same row of the destination field
    const size_t width = (size_t)o_cnt * n_inner * cs;
    cudaStream_t s = (cudaStream_t)stream;
    for (int i = 0; i < P; i++) {
        const int p = (rank + i) % P;                               // every rank starts with a different peer
        const char *srcp = (const char *)send + (size_t)p * rows_per_peer * spitch + (size_t)o0 * n_inner * cs;
        char *dstp = (char *)peer_ptrs_host[p] + (size_t)(outer_start + o0) * n_inner * cs;
        NBK_CUDA(cudaMemcpy2DAsync(dstp, dpitch, srcp, spitch, width, (size_t)rows_per_peer, cudaMemcpyDeviceToDevice, s));
    }
    return NBK_OK;
}

// =============================================================================================
// Mixed-radix path: sides N = 2^a 3^b 5^c 7^d (pmesh / pfft accept any size; nbodykit scripts use 96, 100, 360, 768,
// 1536 ...).  Separate entry points (nbk_r2c_mixed, nbk_c2r_mixed, nbk_fft_lines_mixed, nbk_fft_z_mixed): the
// power-of-two kernels above are untouched.
//   plan     : in-place decimation in frequency over a host-chosen list of radices from {8, 4, 2, 7, 5, 3} (radix 8 while
//              three factors of two remain, then one 4 or 2, then the odd factors), packed 4 bits per stage into one
//              kernel argument.  One register butterfly per radix; 3, 5 and 7 use constant roots.  The output position
//              of frequency k is the mixed-radix digit reversal of k for that plan, tabulated once per CTA in shared
//              memory (ushort[N]).
//   inverse  : IDFT(x)[k] = DFT(x)[(N - k) mod N] -- the store reads the reversed frequency, nothing is conjugated.
//   lines    : k_fft_lines_mixed, the k_fft_lines skeleton (tiles [N][B+1] of B adjacent columns, cp.async double
//              buffering, twiddles W_N^i staged in shared memory, scale folded into the store).
//   z pass   : k_fft_z_mixed, a tile of whole contiguous rows per CTA (lanes along the row).  Even Nz: packed
//              Nz/2-point complex FFT + Hermitian split with W_Nz^k (the inverse combines first).  Odd Nz: two real rows
//              packed as re + i im, one Nz-point FFT, X_a = (Z[k] + conj Z[-k]) / 2, X_b = (Z[k] - conj Z[-k]) / 2i; the
//              inverse rebuilds both Hermitian rows in shared memory while loading.
//   limits   : every complex line is at most 4096 points (Nx, Ny <= 4096; even Nz <= 8192; odd Nz <= 4095): every tile,
//              twiddle table and digit-reversal table then fits in 227 KB of shared memory.
// =============================================================================================
#define NBK_MR_MAX_LINE 4096
#define NBK_MR_MAX_STAGES 16

struct MixedPlan {
    int n;                        // complex points per line
    int nstage;
    unsigned long long radices;   // radix of stage s in bits [4 s, 4 s + 4); stage 0 splits the whole line
};

__device__ __forceinline__ int mr_radix(const MixedPlan &p, int s) { return (int)((p.radices >> (4 * s)) & 15); }

// cos / sin (2 pi h / R) of the odd radices, 1 <= h < R (constant-folded once the butterfly loops are unrolled)
__device__ __forceinline__ double mr_cos(int R, int h) {
    if (h > R / 2) h = R - h;
    if (R == 3) return -0.5;
    if (R == 5) return h == 1 ? 0.30901699437494742410 : -0.80901699437494742410;
    return h == 1 ? 0.62348980185873353053 : (h == 2 ? -0.22252093395631440429 : -0.90096886790241912624);
}
__device__ __forceinline__ double mr_sin(int R, int h) {
    const double sg = h > R / 2 ? -1.0 : 1.0;
    if (h > R / 2) h = R - h;
    if (R == 3) return sg * 0.86602540378443864676;
    if (R == 5) return sg * (h == 1 ? 0.95105651629515357212 : 0.58778525229247312917);
    return sg * (h == 1 ? 0.78183148246802980871 : (h == 2 ? 0.97492791218182360702 : 0.43388373911755812048));
}

// R-point forward DFT, R odd, natural order in and out:  X_m = A_m - i B_m,  X_{R-m} = A_m + i B_m  with
// A_m = a_0 + sum_j cos(2 pi j m / R) (a_j + a_{R-j}),  B_m = sum_j sin(2 pi j m / R) (a_j - a_{R-j}),  j = 1 .. (R-1)/2
template <typename T, typename C, int R>
__device__ __forceinline__ void dft_odd(C (&a)[R]) {
    constexpr int H = (R - 1) / 2;
    C s[H], d[H];
    C x0 = a[0];
#pragma unroll
    for (int j = 1; j <= H; j++) {
        s[j - 1] = cadd(a[j], a[R - j]);
        d[j - 1] = csub(a[j], a[R - j]);
        x0 = cadd(x0, s[j - 1]);
    }
#pragma unroll
    for (int m = 1; m <= H; m++) {
        C A = a[0], Bm = C{0, 0};
#pragma unroll
        for (int j = 1; j <= H; j++) {
            const T c = (T)mr_cos(R, (j * m) % R), sn = (T)mr_sin(R, (j * m) % R);
            A.x += c * s[j - 1].x;
            A.y += c * s[j - 1].y;
            Bm.x += sn * d[j - 1].x;
            Bm.y += sn * d[j - 1].y;
        }
        a[m] = C{A.x + Bm.y, A.y - Bm.x};
        a[R - m] = C{A.x - Bm.y, A.y + Bm.x};
    }
    a[0] = x0;
}

template <typename T, typename C, int R>
__device__ __forceinline__ void dft_mixed(C (&a)[R]) {
    if constexpr (R == 8) radix8(a);
    else if constexpr (R == 4) dft4(a[0], a[1], a[2], a[3]);
    else if constexpr (R == 2) { C x0 = a[0], x1 = a[1]; a[0] = cadd(x0, x1); a[1] = csub(x0, x1); }
    else dft_odd<T, C, R>(a);
}

// tile row pitch: B + 1 elements (conflict-free quarter-warp accesses); a single column needs no padding
template <int B> struct MrPitch { static constexpr int v = B > 1 ? B + 1 : 1; };

// one DIF stage of radix R over B side-by-side lines: sub-transforms of length Ns, Q = Ns / R.  Twiddle
// W_Ns^{q m} = tw[q m (N / Ns) twmul]  (tw is W_{N twmul}^i: twmul = 2 when the table belongs to the unpacked row)
template <typename T, typename C, int B, int R>
__device__ __forceinline__ void mr_stage(C *sm, const C *tw, int N, int Ns, int twmul) {
    constexpr int pitch = MrPitch<B>::v;
    const int Q = Ns / R;
    const int tws = (N / Ns) * twmul;
    const int work = (N / R) * B;
    for (int w = threadIdx.x; w < work; w += blockDim.x) {
        const int b = w % B, t = w / B;
        const int blk = t / Q, q = t - blk * Q;
        C *p = sm + (blk * Ns + q) * pitch + b;
        C a[R];
#pragma unroll
        for (int j = 0; j < R; j++) a[j] = p[j * Q * pitch];
        dft_mixed<T, C, R>(a);
        p[0] = a[0];
        const int ti = q * tws;
#pragma unroll
        for (int m = 1; m < R; m++) p[m * Q * pitch] = ti ? cmul(a[m], tw[m * ti]) : a[m];
    }
    __syncthreads();
}

// in-place forward DIF of B lines held at sm[n * pitch + b]; all threads of the CTA call (it ends with a barrier)
template <typename T, typename C, int B>
__device__ __forceinline__ void mr_fft_tile(C *sm, const C *tw, const MixedPlan &plan, int twmul) {
    int Ns = plan.n;
    for (int s = 0; s < plan.nstage; s++) {
        const int R = mr_radix(plan, s);
        switch (R) {
            case 8: mr_stage<T, C, B, 8>(sm, tw, plan.n, Ns, twmul); break;
            case 4: mr_stage<T, C, B, 4>(sm, tw, plan.n, Ns, twmul); break;
            case 2: mr_stage<T, C, B, 2>(sm, tw, plan.n, Ns, twmul); break;
            case 3: mr_stage<T, C, B, 3>(sm, tw, plan.n, Ns, twmul); break;
            case 5: mr_stage<T, C, B, 5>(sm, tw, plan.n, Ns, twmul); break;
            default: mr_stage<T, C, B, 7>(sm, tw, plan.n, Ns, twmul); break;
        }
        Ns /= R;
    }
}

// position of frequency k after mr_fft_tile (mixed-radix digit reversal)
__device__ __forceinline__ int mr_pos(const MixedPlan &plan, int k) {
    int rem = k, base = plan.n, pos = 0;
    for (int s = 0; s < plan.nstage; s++) {
        const int R = mr_radix(plan, s);
        const int d = rem % R;
        rem /= R;
        base /= R;
        pos += d * base;
    }
    return pos;
}

// perm[k] = mr_pos(plan, k).  No barrier.
__device__ __forceinline__ void mr_build_perm(unsigned short *perm, const MixedPlan &plan) {
    for (int k = threadIdx.x; k < plan.n; k += blockDim.x) perm[k] = (unsigned short)mr_pos(plan, k);
}

// strided tile -> shared [N][pitch] with cp.async; columns beyond the valid width are zero-filled with plain stores
template <typename C, int B>
__device__ __forceinline__ void mr_prefetch_tile(C *sm, const C *base, int N, int64_t line_stride, int bvalid) {
    constexpr int pitch = MrPitch<B>::v;
    for (int w = threadIdx.x; w < N * B; w += blockDim.x) {
        const int b = w % B, n = w / B;
        if (b < bvalid) cp_async_elem(&sm[n * pitch + b], base + (int64_t)n * line_stride + b);
        else sm[n * pitch + b] = C{0, 0};
    }
}

// strided line pass, element(outer, n, inner) = data[outer * outer_stride + n * line_stride + inner].  dst == src: in
// place (a CTA reads its whole tile before it stores any of it).
// shared: buf[2][N][pitch] | W_N^i [N] | perm ushort[N]
template <typename T, int B>
__global__ void __launch_bounds__(512)
k_fft_lines_mixed(const typename C2<T>::type *src, typename C2<T>::type *dst, const typename C2<T>::type *__restrict__ tw_g,
                  MixedPlan plan, int64_t line_stride, int64_t n_inner, int64_t tiles_inner, int64_t n_tiles,
                  int64_t outer_stride, int inverse, T scale) {
    typedef typename C2<T>::type C;
    constexpr int pitch = MrPitch<B>::v;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int N = plan.n;
    C *buf0 = reinterpret_cast<C *>(smem_raw);
    C *buf1 = buf0 + (size_t)N * pitch;
    C *tw = buf1 + (size_t)N * pitch;
    unsigned short *perm = reinterpret_cast<unsigned short *>(tw + N);
    for (int i = threadIdx.x; i < N; i += blockDim.x) tw[i] = tw_g[i];
    mr_build_perm(perm, plan);
    int64_t tile = blockIdx.x;
    if (tile < n_tiles) {
        const int64_t outer = tile / tiles_inner;
        const int64_t inner0 = (tile - outer * tiles_inner) * B;
        const int bvalid = (int)((n_inner - inner0) < B ? (n_inner - inner0) : B);
        mr_prefetch_tile<C, B>(buf0, src + outer * outer_stride + inner0, N, line_stride, bvalid);
    }
    cp_async_commit();
    int cur = 0;
    for (; tile < n_tiles; tile += gridDim.x, cur ^= 1) {
        C *sm = cur ? buf1 : buf0;
        const int64_t outer = tile / tiles_inner;
        const int64_t inner0 = (tile - outer * tiles_inner) * B;
        C *obase = dst + outer * outer_stride + inner0;
        const int bvalid = (int)((n_inner - inner0) < B ? (n_inner - inner0) : B);
        const int64_t nxt = tile + gridDim.x;
        if (nxt < n_tiles) {
            const int64_t o2 = nxt / tiles_inner;
            const int64_t i2 = (nxt - o2 * tiles_inner) * B;
            const int bv2 = (int)((n_inner - i2) < B ? (n_inner - i2) : B);
            mr_prefetch_tile<C, B>(cur ? buf0 : buf1, src + o2 * outer_stride + i2, N, line_stride, bv2);
        }
        cp_async_commit();
        cp_async_wait<1>();          // this tile's copies have landed (the prefetch may still be in flight)
        __syncthreads();             // (the first time through also publishes tw and perm)
        mr_fft_tile<T, C, B>(sm, tw, plan, 1);
        for (int w = threadIdx.x; w < N * B; w += blockDim.x) {
            const int b = w % B, k = w / B;
            if (b < bvalid) {
                const int kk = (inverse && k) ? N - k : k;
                const C v = sm[perm[kk] * pitch + b];
                obase[(int64_t)k * line_stride + b] = C{v.x * scale, v.y * scale};
            }
        }
        __syncthreads();             // everyone is done with `sm` before the next prefetch overwrites it
    }
    cp_async_wait<0>();
}

// z pass: real rows [rows][Nz] <-> complex rows [rows][Nz/2+1].  A tile holds B complex lines of plan.n points: one
// row each (even Nz, n = Nz/2, packed pairs) or two rows each (odd Nz, n = Nz, row 2b in re, row 2b+1 in im).
// shared: tile [n][pitch] | W_Nz^i [Nz] | perm ushort[n].  Forward scaled by `scale`, inverse unnormalised times `scale`.
template <typename T, int B>
__global__ void __launch_bounds__(256)
k_fft_z_mixed(const void *in, void *out, const typename C2<T>::type *__restrict__ tw_g, MixedPlan plan, int Nz,
              int64_t rows, int inverse, T scale) {
    typedef typename C2<T>::type C;
    constexpr int pitch = MrPitch<B>::v;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int L = plan.n;
    const bool odd = Nz & 1;
    const int Nzc = Nz / 2 + 1;
    const int rpl = odd ? 2 : 1;                   // real rows per complex line
    C *sm = reinterpret_cast<C *>(smem_raw);
    C *tw = sm + (size_t)L * pitch;
    unsigned short *perm = reinterpret_cast<unsigned short *>(tw + Nz);
    for (int i = threadIdx.x; i < Nz; i += blockDim.x) tw[i] = tw_g[i];
    mr_build_perm(perm, plan);
    __syncthreads();
    const int64_t per_tile = (int64_t)B * rpl;
    const int64_t n_tiles = (rows + per_tile - 1) / per_tile;
    const T h = (T)0.5 * scale;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t row0 = tile * per_tile;
        const int nrows = (int)((rows - row0) < per_tile ? (rows - row0) : per_tile);
        // ---- load (lanes along the contiguous rows)
        if (!inverse && !odd) {
            const C *src = reinterpret_cast<const C *>(static_cast<const T *>(in) + row0 * Nz);
            for (int w = threadIdx.x; w < L * B; w += blockDim.x) {
                const int b = w / L, n = w - b * L;
                sm[n * pitch + b] = b < nrows ? src[(int64_t)b * L + n] : C{0, 0};
            }
        } else if (!inverse) {
            const T *src = static_cast<const T *>(in) + row0 * Nz;
            for (int w = threadIdx.x; w < L * B; w += blockDim.x) {
                const int b = w / L, n = w - b * L;
                const T xa = 2 * b < nrows ? src[(int64_t)(2 * b) * Nz + n] : (T)0;
                const T xb = 2 * b + 1 < nrows ? src[(int64_t)(2 * b + 1) * Nz + n] : (T)0;
                sm[n * pitch + b] = C{xa, xb};
            }
        } else if (!odd) {
            // Z[k] = E + i O,  E = X[k] + conj X[M-k],  O = conj(W_Nz^k) (X[k] - conj X[M-k]),  k < M  (the factor 1/2 of
            // the split and the 2 of the unnormalised inverse cancel)
            const C *src = static_cast<const C *>(in) + row0 * Nzc;
            for (int w = threadIdx.x; w < L * B; w += blockDim.x) {
                const int b = w / L, k = w - b * L;
                C z = C{0, 0};
                if (b < nrows) {
                    C xk = src[(int64_t)b * Nzc + k];
                    C xm = cconj(src[(int64_t)b * Nzc + (L - k)]);
                    if (k == 0) { xk.y = 0; xm.y = 0; }     // the k = 0 and k = Nz/2 modes of a real row are real
                    const C e = cadd(xk, xm), d = csub(xk, xm);
                    const C o = cmul(cconj(tw[k]), d);
                    z = C{e.x - o.y, e.y + o.x};
                }
                sm[k * pitch + b] = z;
            }
        } else {
            // both Hermitian rows rebuilt in the tile: Z[k] = X_a[k] + i X_b[k], Z[Nz-k] = conj X_a[k] + i conj X_b[k]
            const C *src = static_cast<const C *>(in) + row0 * Nzc;
            for (int w = threadIdx.x; w < Nzc * B; w += blockDim.x) {
                const int b = w / Nzc, k = w - b * Nzc;
                C A = 2 * b < nrows ? src[(int64_t)(2 * b) * Nzc + k] : C{0, 0};
                C Bv = 2 * b + 1 < nrows ? src[(int64_t)(2 * b + 1) * Nzc + k] : C{0, 0};
                if (k == 0) { A.y = 0; Bv.y = 0; }          // the k = 0 mode of a real row is real
                sm[k * pitch + b] = C{A.x - Bv.y, A.y + Bv.x};
                if (k) sm[(L - k) * pitch + b] = C{A.x + Bv.y, Bv.x - A.y};
            }
        }
        __syncthreads();
        mr_fft_tile<T, C, B>(sm, tw, plan, odd ? 1 : 2);
        // ---- store
        if (!inverse && !odd) {
            // X[k] = 1/2 [ (Z[k] + conj Z[M-k]) - i W_Nz^k (Z[k] - conj Z[M-k]) ],  k = 0 .. M  (Z[M] := Z[0])
            C *dst = static_cast<C *>(out) + row0 * Nzc;
            for (int w = threadIdx.x; w < Nzc * B; w += blockDim.x) {
                const int b = w / Nzc, k = w - b * Nzc;
                if (b < nrows) {
                    const C zk = sm[perm[k == L ? 0 : k] * pitch + b];
                    const C zm = cconj(sm[perm[k == 0 ? 0 : L - k] * pitch + b]);
                    const C e = cadd(zk, zm), o = csub(zk, zm);
                    const C wo = cmul(tw[k], o);
                    dst[(int64_t)b * Nzc + k] = C{(e.x + wo.y) * h, (e.y - wo.x) * h};
                }
            }
        } else if (!inverse) {
            // X_a[k] = (Z[k] + conj Z[-k]) / 2,  X_b[k] = -i (Z[k] - conj Z[-k]) / 2
            C *dst = static_cast<C *>(out) + row0 * Nzc;
            for (int w = threadIdx.x; w < Nzc * B; w += blockDim.x) {
                const int b = w / Nzc, k = w - b * Nzc;
                if (2 * b < nrows) {
                    const C zk = sm[perm[k] * pitch + b];
                    const C zm = cconj(sm[perm[k ? L - k : 0] * pitch + b]);
                    const C e = cadd(zk, zm), d = csub(zk, zm);
                    dst[(int64_t)(2 * b) * Nzc + k] = C{e.x * h, e.y * h};
                    if (2 * b + 1 < nrows) dst[(int64_t)(2 * b + 1) * Nzc + k] = C{d.y * h, -d.x * h};
                }
            }
        } else if (!odd) {
            // x[2n] + i x[2n+1] = sum_k Z[k] e^{+2 pi i k n / M} = DFT(Z)[(M - n) mod M]
            C *dst = reinterpret_cast<C *>(static_cast<T *>(out) + row0 * Nz);
            for (int w = threadIdx.x; w < L * B; w += blockDim.x) {
                const int b = w / L, n = w - b * L;
                if (b < nrows) {
                    const C v = sm[perm[n ? L - n : 0] * pitch + b];
                    dst[(int64_t)b * L + n] = C{v.x * scale, v.y * scale};
                }
            }
        } else {
            T *dst = static_cast<T *>(out) + row0 * Nz;
            for (int w = threadIdx.x; w < L * B; w += blockDim.x) {
                const int b = w / L, n = w - b * L;
                if (2 * b < nrows) {
                    const C v = sm[perm[n ? L - n : 0] * pitch + b];
                    dst[(int64_t)(2 * b) * Nz + n] = v.x * scale;
                    if (2 * b + 1 < nrows) dst[(int64_t)(2 * b + 1) * Nz + n] = v.y * scale;
                }
            }
        }
        __syncthreads();
    }
}

// ---- host side
static bool is_7smooth(int64_t n) {
    if (n < 1) return false;
    for (int p : {2, 3, 5, 7})
        while (n % p == 0) n /= p;
    return n == 1;
}

static MixedPlan mr_plan(int n) {
    MixedPlan p;
    p.n = n;
    p.nstage = 0;
    p.radices = 0;
    auto push = [&](int r) { p.radices |= (unsigned long long)r << (4 * p.nstage); p.nstage++; };
    int m = n, c2 = 0;
    while (m % 2 == 0) { m /= 2; c2++; }
    for (; c2 >= 3; c2 -= 3) push(8);
    if (c2 == 2) push(4);
    else if (c2 == 1) push(2);
    for (int r : {7, 5, 3})
        while (m % r == 0) { m /= r; push(r); }
    return p;
}

// complex line length n (2 .. 4096, 7-smooth)
static int check_line_mixed(const char *who, int64_t n) {
    NBK_CHECK_ARG(n >= 2 && n <= NBK_MR_MAX_LINE && is_7smooth(n),
                  "%s: line length %lld unsupported: the mixed-radix FFT takes lengths 2 .. 4096 whose prime factors are "
                  "2, 3, 5 and 7", who, (long long)n);
    return NBK_OK;
}

static int check_z_mixed(const char *who, int64_t Nz) {
    NBK_CHECK_ARG(Nz >= 2 && is_7smooth(Nz) && ((Nz % 2 == 0 && Nz <= 2 * NBK_MR_MAX_LINE) || (Nz % 2 && Nz < NBK_MR_MAX_LINE)),
                  "%s: Nz = %lld unsupported: the mixed-radix z pass takes 7-smooth lengths (prime factors 2, 3, 5, 7), "
                  "even up to 8192 or odd up to 4095", who, (long long)Nz);
    return NBK_OK;
}

static int check_dims_mixed(const char *who, int dtype, const int64_t *nmesh) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "%s: bad dtype %d", who, dtype);
    const int64_t Nx = nmesh[0], Ny = nmesh[1], Nz = nmesh[2];
    const bool zok = Nz >= 2 && is_7smooth(Nz) && ((Nz % 2 == 0 && Nz <= 2 * NBK_MR_MAX_LINE) || (Nz % 2 && Nz < NBK_MR_MAX_LINE));
    NBK_CHECK_ARG(Nx >= 2 && Ny >= 2 && Nx <= NBK_MR_MAX_LINE && Ny <= NBK_MR_MAX_LINE && is_7smooth(Nx) && is_7smooth(Ny) && zok,
                  "%s: Nmesh (%lld,%lld,%lld) unsupported: each side must be a product of 2, 3, 5 and 7 (Nx, Ny 2 .. 4096; "
                  "Nz 2 .. 8192 if even, up to 4095 if odd)", who, (long long)Nx, (long long)Ny, (long long)Nz);
    return NBK_OK;
}

template <typename T>
static int launch_lines_mixed(const void *src, void *dst, int N, int64_t line_stride, int64_t n_inner, int64_t n_outer,
                              int64_t outer_stride, int inverse, double scale, cudaStream_t s) {
    typedef typename C2<T>::type C;
    const int dtype = sizeof(T) == 4 ? NBK_F4 : NBK_F8;
    void *tw;
    int rc = get_twiddle(N, dtype, s, &tw);
    if (rc) return rc;
    // two tile buffers + twiddles + digit-reversal table; 128-byte runs while that fits, narrower for long lines
    auto smem_for = [&](int B) { return (size_t)N * (2 * (B > 1 ? B + 1 : 1) + 1) * sizeof(C) + (size_t)N * 2 + 16; };
    int B = 128 / (int)sizeof(C);
    while (B > 1 && (smem_for(B) > 220 * 1024 || B / 2 >= n_inner)) B >>= 1;
    const size_t smem = smem_for(B);
    NBK_CHECK_ARG(smem <= 227 * 1024, "fft_lines_mixed: N=%d does not fit in shared memory", N);
    const int64_t tiles_inner = (n_inner + B - 1) / B;
    const int64_t n_tiles = tiles_inner * n_outer;
    int per_sm = (int)((227 * 1024) / (smem + 1024));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 8) per_sm = 8;
    const int64_t g = n_tiles < (int64_t)NBK_SM_COUNT * per_sm ? n_tiles : (int64_t)NBK_SM_COUNT * per_sm;
    const int nthreads = (per_sm == 1 && (int64_t)N * B >= 4096) ? 512 : 256;
    const MixedPlan plan = mr_plan(N);
#define LAUNCH_LM(BB)                                                                                              \
    case BB:                                                                                                       \
        NBK_CUDA(cudaFuncSetAttribute(k_fft_lines_mixed<T, BB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        k_fft_lines_mixed<T, BB><<<(int)g, nthreads, smem, s>>>((const C *)src, (C *)dst, (const C *)tw, plan, line_stride, \
                                                                 n_inner, tiles_inner, n_tiles, outer_stride, inverse, (T)scale); \
        break;
    switch (B) {
        LAUNCH_LM(1) LAUNCH_LM(2) LAUNCH_LM(4) LAUNCH_LM(8) LAUNCH_LM(16)
        default: nbk_set_error("fft_lines_mixed: internal tile width %d", B); return NBK_ERR_ARG;
    }
#undef LAUNCH_LM
    NBK_LAUNCHED();
    return NBK_OK;
}

template <typename T>
static int launch_z_mixed(const void *in, void *out, int64_t rows, int Nz, int inverse, double scale, cudaStream_t s) {
    typedef typename C2<T>::type C;
    const int dtype = sizeof(T) == 4 ? NBK_F4 : NBK_F8;
    void *tw;
    int rc = get_twiddle(Nz, dtype, s, &tw);
    if (rc) return rc;
    const bool odd = Nz & 1;
    const int L = odd ? Nz : Nz / 2;
    const int64_t lines = odd ? (rows + 1) / 2 : rows;
    // B rows per tile: as many as leave two CTAs per SM (one CTA's loads overlap the other's butterflies); long rows
    // take the whole SM
    auto smem_for = [&](int B) { return ((size_t)L * (B > 1 ? B + 1 : 1) + Nz) * sizeof(C) + (size_t)L * 2 + 16; };
    int B = 16;
    while (B > 1 && (smem_for(B) > 110 * 1024 || B / 2 >= lines)) B >>= 1;
    const size_t smem = smem_for(B);
    NBK_CHECK_ARG(smem <= 227 * 1024, "fft_z_mixed: Nz=%d does not fit in shared memory", Nz);
    const int64_t n_tiles = (lines + B - 1) / B;
    int per_sm = (int)((227 * 1024) / (smem + 1024));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 8) per_sm = 8;
    const int64_t g = n_tiles < (int64_t)NBK_SM_COUNT * per_sm ? n_tiles : (int64_t)NBK_SM_COUNT * per_sm;
    const MixedPlan plan = mr_plan(L);
#define LAUNCH_ZM(BB)                                                                                              \
    case BB:                                                                                                       \
        NBK_CUDA(cudaFuncSetAttribute(k_fft_z_mixed<T, BB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        k_fft_z_mixed<T, BB><<<(int)g, 256, smem, s>>>(in, out, (const C *)tw, plan, Nz, rows, inverse, (T)scale); \
        break;
    switch (B) {
        LAUNCH_ZM(1) LAUNCH_ZM(2) LAUNCH_ZM(4) LAUNCH_ZM(8) LAUNCH_ZM(16)
        default: nbk_set_error("fft_z_mixed: internal tile width %d", B); return NBK_ERR_ARG;
    }
#undef LAUNCH_ZM
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_fft_lines_mixed(const void *src, void *dst, int dtype, int64_t n_line, int64_t line_stride, int64_t n_inner,
                                   int64_t n_outer, int64_t outer_stride, int inverse, double scale, void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "fft_lines_mixed: bad dtype %d", dtype);
    int rc = check_line_mixed("fft_lines_mixed", n_line);
    if (rc) return rc;
    if (n_inner <= 0 || n_outer <= 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == NBK_F4)
        return launch_lines_mixed<float>(src, dst, (int)n_line, line_stride, n_inner, n_outer, outer_stride, inverse, scale, s);
    return launch_lines_mixed<double>(src, dst, (int)n_line, line_stride, n_inner, n_outer, outer_stride, inverse, scale, s);
}

extern "C" int nbk_fft_z_mixed(const void *in, void *out, int dtype, int64_t rows, int64_t Nz, int inverse, double scale,
                               void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "fft_z_mixed: bad dtype %d", dtype);
    int rc = check_z_mixed("fft_z_mixed", Nz);
    if (rc) return rc;
    if (rows <= 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    return (dtype == NBK_F4) ? launch_z_mixed<float>(in, out, rows, (int)Nz, inverse, scale, s)
                             : launch_z_mixed<double>(in, out, rows, (int)Nz, inverse, scale, s);
}

extern "C" int nbk_r2c_mixed(const void *real, void *cplx, int dtype, const int64_t *nmesh, double extra_scale, void *stream) {
    int rc = check_dims_mixed("r2c_mixed", dtype, nmesh);
    if (rc) return rc;
    const int64_t Nx = nmesh[0], Ny = nmesh[1], Nz = nmesh[2], Nzc = Nz / 2 + 1;
    rc = nbk_fft_z_mixed(real, cplx, dtype, Nx * Ny, Nz, 0, 1.0, stream);
    if (rc) return rc;
    rc = nbk_fft_lines_mixed(cplx, cplx, dtype, Ny, Nzc, Nzc, Nx, Ny * Nzc, 0, 1.0, stream);
    if (rc) return rc;
    const double scale = extra_scale / ((double)Nx * (double)Ny * (double)Nz);
    return nbk_fft_lines_mixed(cplx, cplx, dtype, Nx, Ny * Nzc, Ny * Nzc, 1, 0, 0, scale, stream);
}

// c2r destroys its complex input unless `work` (same size as cplx) is given
extern "C" int nbk_c2r_mixed(const void *cplx, void *real, int dtype, const int64_t *nmesh, void *work, void *stream) {
    int rc = check_dims_mixed("c2r_mixed", dtype, nmesh);
    if (rc) return rc;
    const int64_t Nx = nmesh[0], Ny = nmesh[1], Nz = nmesh[2], Nzc = Nz / 2 + 1;
    void *c = const_cast<void *>(cplx);
    if (work && work != cplx) {
        const size_t bytes = (size_t)Nx * Ny * Nzc * (dtype == NBK_F4 ? 8 : 16);
        NBK_CUDA(cudaMemcpyAsync(work, cplx, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
        c = work;
    }
    rc = nbk_fft_lines_mixed(c, c, dtype, Nx, Ny * Nzc, Ny * Nzc, 1, 0, 1, 1.0, stream);
    if (rc) return rc;
    rc = nbk_fft_lines_mixed(c, c, dtype, Ny, Nzc, Nzc, Nx, Ny * Nzc, 1, 1.0, stream);
    if (rc) return rc;
    return nbk_fft_z_mixed(c, real, dtype, Nx * Ny, Nz, 1, 1.0, stream);
}

// =============================================================================================
// Bluestein path: lines whose length has a prime factor above 7 (pmesh / pfft hand every side to FFTW; a 1380 box at a
// 5-unit cell gives 276 = 2^2 3 23).  Separate entry points (nbk_fft_lines_bluestein, nbk_fft_z_bluestein) with the
// argument lists and limits of the mixed-radix pair; ParticleMesh picks them per axis.
//   identity : nk = (n^2 + k^2 - (k - n)^2) / 2, so with the chirp c[n] = e^{i pi n^2 / N}
//              X[k] = conj c[k] sum_n (x[n] conj c[n]) c[k - n], a cyclic convolution of length M, the smallest 7-smooth
//              number >= 2N - 1, which the mixed-radix stages transform.
//   tile     : B lines of M points in shared memory, [M][pitch] as in k_fft_lines_mixed.  a = x conj c, zero-padded to M;
//              forward DIF (mr_fft_tile, digit-reversed output); times the filter spectrum FFT(c) / M, tabulated in the
//              same digit-reversed order; then the transposed network (mr_fft_tile_dit: the DIT stages in reverse order
//              take digit-reversed input to natural output) gives the forward DFT F in natural order, and the
//              convolution is y[k] = F[(M - k) mod M].  No digit-reversal table, no second M-point buffer.
//   inverse  : IDFT(x)[k] = DFT(x)[(N - k) mod N], as in the mixed path.
//   tables   : per (N, dtype), cached with the twiddles: conj c[n] (phase from n^2 mod 2N in 64-bit integers, sincospi in
//              f8) and the filter spectrum (a direct f8 sum of N terms per frequency), rounded to f4 only at the end.
//              W_M sits in shared memory when it fits beside the tile, else it is read through L2 (f8 at M = 8192: the
//              one-line tile alone is 128 KB); chirp and filter are always read through L2.
//   limits   : the mixed path's: complex lines of 2 .. 4096 points (M <= 8192), even Nz <= 8192, odd Nz <= 4095.
// =============================================================================================

// one DIT stage, the transpose of mr_stage (twiddles first, then the radix-R DFT: both matrices are symmetric)
template <typename T, typename C, int B, int R>
__device__ __forceinline__ void mr_stage_dit(C *sm, const C *tw, int N, int Ns) {
    constexpr int pitch = MrPitch<B>::v;
    const int Q = Ns / R;
    const int tws = N / Ns;
    const int work = (N / R) * B;
    for (int w = threadIdx.x; w < work; w += blockDim.x) {
        const int b = w % B, t = w / B;
        const int blk = t / Q, q = t - blk * Q;
        C *p = sm + (blk * Ns + q) * pitch + b;
        const int ti = q * tws;
        C a[R];
        a[0] = p[0];
#pragma unroll
        for (int m = 1; m < R; m++) a[m] = ti ? cmul(p[m * Q * pitch], tw[m * ti]) : p[m * Q * pitch];
        dft_mixed<T, C, R>(a);
#pragma unroll
        for (int j = 0; j < R; j++) p[j * Q * pitch] = a[j];
    }
    __syncthreads();
}

// forward DFT of B lines held in the digit-reversed order mr_fft_tile leaves, into natural order: the stages of
// mr_fft_tile transposed, last first.  All threads of the CTA call (it ends with a barrier).
template <typename T, typename C, int B>
__device__ __forceinline__ void mr_fft_tile_dit(C *sm, const C *tw, const MixedPlan &plan) {
    int Ns = 1;
    for (int s = plan.nstage - 1; s >= 0; s--) {
        const int R = mr_radix(plan, s);
        Ns *= R;
        switch (R) {
            case 8: mr_stage_dit<T, C, B, 8>(sm, tw, plan.n, Ns); break;
            case 4: mr_stage_dit<T, C, B, 4>(sm, tw, plan.n, Ns); break;
            case 2: mr_stage_dit<T, C, B, 2>(sm, tw, plan.n, Ns); break;
            case 3: mr_stage_dit<T, C, B, 3>(sm, tw, plan.n, Ns); break;
            case 5: mr_stage_dit<T, C, B, 5>(sm, tw, plan.n, Ns); break;
            default: mr_stage_dit<T, C, B, 7>(sm, tw, plan.n, Ns); break;
        }
    }
}

// N-point forward DFT of B lines by Bluestein's identity, plan = mr_plan(M), tw = W_M^i.  On entry sm[n * pitch + b],
// n < N, holds the input (published by a barrier); on exit sm[k * pitch + b], k < N, holds the unscaled DFT in
// natural order.  All threads of the CTA call (it ends with a barrier).
template <typename T, typename C, int B>
__device__ __forceinline__ void bs_fft_tile(C *sm, const C *tw, const C *__restrict__ chirp, const C *__restrict__ filt,
                                            const MixedPlan &plan, int N) {
    constexpr int pitch = MrPitch<B>::v;
    const int M = plan.n;
    for (int w = threadIdx.x; w < M * B; w += blockDim.x) {
        const int b = w % B, n = w / B;
        sm[n * pitch + b] = n < N ? cmul(sm[n * pitch + b], chirp[n]) : C{0, 0};
    }
    __syncthreads();
    mr_fft_tile<T, C, B>(sm, tw, plan, 1);
    for (int w = threadIdx.x; w < M * B; w += blockDim.x) {
        const int b = w % B, n = w / B;
        sm[n * pitch + b] = cmul(sm[n * pitch + b], filt[n]);
    }
    __syncthreads();
    mr_fft_tile_dit<T, C, B>(sm, tw, plan);
    // y[k] = F[(M - k) mod M]: for k > 0 it lies at M - k >= N (M >= 2N - 1), so no write meets another thread's read
    for (int w = threadIdx.x; w < N * B; w += blockDim.x) {
        const int b = w % B, k = w / B;
        sm[k * pitch + b] = cmul(sm[(k ? M - k : 0) * pitch + b], chirp[k]);
    }
    __syncthreads();
}

// stage W_M^i in shared memory after the tile when the launch made room for it; otherwise read it through L2
template <typename C>
__device__ __forceinline__ const C *bs_twiddles(C *smtw, const C *tw_g, int M, int tw_shared) {
    if (!tw_shared) return tw_g;
    for (int i = threadIdx.x; i < M; i += blockDim.x) smtw[i] = tw_g[i];
    return smtw;
}

// strided line pass with the contract of k_fft_lines_mixed: element(outer, n, inner), dst == src in place (a CTA reads
// its whole tile before it stores any of it), scale folded into the store.  shared: tile [M][pitch] | W_M^i [M]
template <typename T, int B>
__global__ void __launch_bounds__(512, 1)
k_fft_lines_bluestein(const typename C2<T>::type *src, typename C2<T>::type *dst, const typename C2<T>::type *__restrict__ tw_g,
                      const typename C2<T>::type *__restrict__ chirp, const typename C2<T>::type *__restrict__ filt,
                      MixedPlan plan, int N, int64_t line_stride, int64_t n_inner, int64_t tiles_inner, int64_t n_tiles,
                      int64_t outer_stride, int inverse, T scale, int tw_shared) {
    typedef typename C2<T>::type C;
    constexpr int pitch = MrPitch<B>::v;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    C *sm = reinterpret_cast<C *>(smem_raw);
    const C *tw = bs_twiddles<C>(sm + (size_t)plan.n * pitch, tw_g, plan.n, tw_shared);
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t outer = tile / tiles_inner;
        const int64_t inner0 = (tile - outer * tiles_inner) * B;
        const int bvalid = (int)((n_inner - inner0) < B ? (n_inner - inner0) : B);
        const C *ibase = src + outer * outer_stride + inner0;
        for (int w = threadIdx.x; w < N * B; w += blockDim.x) {
            const int b = w % B, n = w / B;
            sm[n * pitch + b] = b < bvalid ? ibase[(int64_t)n * line_stride + b] : C{0, 0};
        }
        __syncthreads();             // (the first time through also publishes tw)
        bs_fft_tile<T, C, B>(sm, tw, chirp, filt, plan, N);
        C *obase = dst + outer * outer_stride + inner0;
        for (int w = threadIdx.x; w < N * B; w += blockDim.x) {
            const int b = w % B, k = w / B;
            if (b < bvalid) {
                const C v = sm[((inverse && k) ? N - k : k) * pitch + b];
                obase[(int64_t)k * line_stride + b] = C{v.x * scale, v.y * scale};
            }
        }
        __syncthreads();             // everyone is done with the tile before the next load overwrites it
    }
}

// z pass with the packing of k_fft_z_mixed: real rows [rows][Nz] <-> complex rows [rows][Nz/2+1]; a tile holds B complex
// lines of L points, one row each (even Nz, L = Nz/2) or two rows each (odd Nz, L = Nz), transformed by Bluestein over
// plan = mr_plan(M).  twz = W_Nz^i (the Hermitian split of even rows, read through L2).  shared: tile [M][pitch] | W_M^i
template <typename T, int B>
__global__ void __launch_bounds__(256)
k_fft_z_bluestein(const void *in, void *out, const typename C2<T>::type *__restrict__ twz,
                  const typename C2<T>::type *__restrict__ tw_g, const typename C2<T>::type *__restrict__ chirp,
                  const typename C2<T>::type *__restrict__ filt, MixedPlan plan, int Nz, int64_t rows, int inverse, T scale,
                  int tw_shared) {
    typedef typename C2<T>::type C;
    constexpr int pitch = MrPitch<B>::v;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const bool odd = Nz & 1;
    const int L = odd ? Nz : Nz / 2;
    const int Nzc = Nz / 2 + 1;
    const int rpl = odd ? 2 : 1;                   // real rows per complex line
    C *sm = reinterpret_cast<C *>(smem_raw);
    const C *tw = bs_twiddles<C>(sm + (size_t)plan.n * pitch, tw_g, plan.n, tw_shared);
    const int64_t per_tile = (int64_t)B * rpl;
    const int64_t n_tiles = (rows + per_tile - 1) / per_tile;
    const T h = (T)0.5 * scale;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t row0 = tile * per_tile;
        const int nrows = (int)((rows - row0) < per_tile ? (rows - row0) : per_tile);
        // ---- load (lanes along the contiguous rows)
        if (!inverse && !odd) {
            const C *src = reinterpret_cast<const C *>(static_cast<const T *>(in) + row0 * Nz);
            for (int w = threadIdx.x; w < L * B; w += blockDim.x) {
                const int b = w / L, n = w - b * L;
                sm[n * pitch + b] = b < nrows ? src[(int64_t)b * L + n] : C{0, 0};
            }
        } else if (!inverse) {
            const T *src = static_cast<const T *>(in) + row0 * Nz;
            for (int w = threadIdx.x; w < L * B; w += blockDim.x) {
                const int b = w / L, n = w - b * L;
                const T xa = 2 * b < nrows ? src[(int64_t)(2 * b) * Nz + n] : (T)0;
                const T xb = 2 * b + 1 < nrows ? src[(int64_t)(2 * b + 1) * Nz + n] : (T)0;
                sm[n * pitch + b] = C{xa, xb};
            }
        } else if (!odd) {
            // Z[k] = E + i O,  E = X[k] + conj X[L-k],  O = conj(W_Nz^k) (X[k] - conj X[L-k]),  k < L
            const C *src = static_cast<const C *>(in) + row0 * Nzc;
            for (int w = threadIdx.x; w < L * B; w += blockDim.x) {
                const int b = w / L, k = w - b * L;
                C z = C{0, 0};
                if (b < nrows) {
                    C xk = src[(int64_t)b * Nzc + k];
                    C xm = cconj(src[(int64_t)b * Nzc + (L - k)]);
                    if (k == 0) { xk.y = 0; xm.y = 0; }     // the k = 0 and k = Nz/2 modes of a real row are real
                    const C e = cadd(xk, xm), d = csub(xk, xm);
                    const C o = cmul(cconj(twz[k]), d);
                    z = C{e.x - o.y, e.y + o.x};
                }
                sm[k * pitch + b] = z;
            }
        } else {
            // both Hermitian rows rebuilt in the tile: Z[k] = X_a[k] + i X_b[k], Z[Nz-k] = conj X_a[k] + i conj X_b[k]
            const C *src = static_cast<const C *>(in) + row0 * Nzc;
            for (int w = threadIdx.x; w < Nzc * B; w += blockDim.x) {
                const int b = w / Nzc, k = w - b * Nzc;
                C A = 2 * b < nrows ? src[(int64_t)(2 * b) * Nzc + k] : C{0, 0};
                C Bv = 2 * b + 1 < nrows ? src[(int64_t)(2 * b + 1) * Nzc + k] : C{0, 0};
                if (k == 0) { A.y = 0; Bv.y = 0; }          // the k = 0 mode of a real row is real
                sm[k * pitch + b] = C{A.x - Bv.y, A.y + Bv.x};
                if (k) sm[(L - k) * pitch + b] = C{A.x + Bv.y, Bv.x - A.y};
            }
        }
        __syncthreads();
        bs_fft_tile<T, C, B>(sm, tw, chirp, filt, plan, L);
        // ---- store (the tile is in natural order)
        if (!inverse && !odd) {
            // X[k] = 1/2 [ (Z[k] + conj Z[L-k]) - i W_Nz^k (Z[k] - conj Z[L-k]) ],  k = 0 .. L  (Z[L] := Z[0])
            C *dst = static_cast<C *>(out) + row0 * Nzc;
            for (int w = threadIdx.x; w < Nzc * B; w += blockDim.x) {
                const int b = w / Nzc, k = w - b * Nzc;
                if (b < nrows) {
                    const C zk = sm[(k == L ? 0 : k) * pitch + b];
                    const C zm = cconj(sm[(k == 0 ? 0 : L - k) * pitch + b]);
                    const C e = cadd(zk, zm), o = csub(zk, zm);
                    const C wo = cmul(twz[k], o);
                    dst[(int64_t)b * Nzc + k] = C{(e.x + wo.y) * h, (e.y - wo.x) * h};
                }
            }
        } else if (!inverse) {
            // X_a[k] = (Z[k] + conj Z[-k]) / 2,  X_b[k] = -i (Z[k] - conj Z[-k]) / 2
            C *dst = static_cast<C *>(out) + row0 * Nzc;
            for (int w = threadIdx.x; w < Nzc * B; w += blockDim.x) {
                const int b = w / Nzc, k = w - b * Nzc;
                if (2 * b < nrows) {
                    const C zk = sm[k * pitch + b];
                    const C zm = cconj(sm[(k ? L - k : 0) * pitch + b]);
                    const C e = cadd(zk, zm), d = csub(zk, zm);
                    dst[(int64_t)(2 * b) * Nzc + k] = C{e.x * h, e.y * h};
                    if (2 * b + 1 < nrows) dst[(int64_t)(2 * b + 1) * Nzc + k] = C{d.y * h, -d.x * h};
                }
            }
        } else if (!odd) {
            // x[2n] + i x[2n+1] = sum_k Z[k] e^{+2 pi i k n / L} = DFT(Z)[(L - n) mod L]
            C *dst = reinterpret_cast<C *>(static_cast<T *>(out) + row0 * Nz);
            for (int w = threadIdx.x; w < L * B; w += blockDim.x) {
                const int b = w / L, n = w - b * L;
                if (b < nrows) {
                    const C v = sm[(n ? L - n : 0) * pitch + b];
                    dst[(int64_t)b * L + n] = C{v.x * scale, v.y * scale};
                }
            }
        } else {
            T *dst = static_cast<T *>(out) + row0 * Nz;
            for (int w = threadIdx.x; w < L * B; w += blockDim.x) {
                const int b = w / L, n = w - b * L;
                if (2 * b < nrows) {
                    const C v = sm[(n ? L - n : 0) * pitch + b];
                    dst[(int64_t)(2 * b) * Nz + n] = v.x * scale;
                    if (2 * b + 1 < nrows) dst[(int64_t)(2 * b + 1) * Nz + n] = v.y * scale;
                }
            }
        }
        __syncthreads();
    }
}

// chirp[n] = conj c[n] = e^{-i pi n^2 / N}; the phase is reduced exactly (n^2 mod 2N) before sincospi
template <typename T>
__global__ void k_bs_chirp(typename C2<T>::type *chirp, int N) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n < N) {
        double s, c;
        sincospi((double)(((int64_t)n * n) % (2 * (int64_t)N)) / (double)N, &s, &c);
        chirp[n].x = (T)c;
        chirp[n].y = (T)-s;
    }
}

// filt[mr_pos(plan, k)] = FFT(b)[k] / M for the filter b[m] = b[M - m] = c[m] (m < N), zero between.  b is even, so
// FFT(b)[k] = 1 + 2 sum_{m=1}^{N-1} c[m] cos(2 pi m k / M): one warp per frequency, f8 throughout.
template <typename T>
__global__ void k_bs_filter(typename C2<T>::type *filt, int N, MixedPlan plan) {
    const int M = plan.n;
    const int lane = threadIdx.x & 31;
    const int64_t k = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (k >= M) return;                            // (whole warps)
    double re = 0.0, im = 0.0;
    for (int m = 1 + lane; m < N; m += 32) {
        double s, c;
        sincospi((double)(((int64_t)m * m) % (2 * (int64_t)N)) / (double)N, &s, &c);
        const double ck = cospi(2.0 * (double)((m * k) % M) / (double)M);
        re += c * ck;
        im += s * ck;
    }
    for (int o = 16; o; o >>= 1) {
        re += __shfl_xor_sync(0xffffffffu, re, o);
        im += __shfl_xor_sync(0xffffffffu, im, o);
    }
    if (lane == 0) {
        typename C2<T>::type v;
        v.x = (T)((1.0 + 2.0 * re) / M);
        v.y = (T)(2.0 * im / M);
        filt[mr_pos(plan, (int)k)] = v;
    }
}

// convolution length of an n-point Bluestein transform: the smallest 7-smooth M >= 2n - 1
static int bs_len(int n) {
    int m = 2 * n - 1;
    while (!is_7smooth(m)) m++;
    return m;
}

// chirp [N] followed by the filter spectrum [M], one allocation per (device, N, dtype), kept in the twiddle map under
// the dtype code + NBK_BS_KEY
#define NBK_BS_KEY 1000
static int get_bluestein(int N, int dtype, cudaStream_t s, void **chirp, void **filt) {
    const int M = bs_len(N);
    const size_t cs = dtype == NBK_F4 ? 8 : 16;
    int dev = 0;
    NBK_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(g_tw_mutex);
    auto key = std::make_tuple(dev, N, dtype + NBK_BS_KEY);
    auto it = g_tw.find(key);
    void *p = nullptr;
    if (it != g_tw.end()) {
        p = it->second;
    } else {
        NBK_CUDA(cudaMalloc(&p, (size_t)(N + M) * cs));
        void *f = (char *)p + (size_t)N * cs;
        const MixedPlan plan = mr_plan(M);
        const int gc = (N + 255) / 256, gf = (M + 7) / 8;     // filter: 8 warps per block
        if (dtype == NBK_F4) k_bs_chirp<float><<<gc, 256, 0, s>>>((float2 *)p, N);
        else k_bs_chirp<double><<<gc, 256, 0, s>>>((double2 *)p, N);
        NBK_LAUNCHED();
        if (dtype == NBK_F4) k_bs_filter<float><<<gf, 256, 0, s>>>((float2 *)f, N, plan);
        else k_bs_filter<double><<<gf, 256, 0, s>>>((double2 *)f, N, plan);
        NBK_LAUNCHED();
        // the tables must be visible to later launches on other streams as well
        NBK_CUDA(cudaStreamSynchronize(s));
        g_tw[key] = p;
    }
    *chirp = p;
    *filt = (char *)p + (size_t)N * cs;
    return NBK_OK;
}

// complex line length n: 2 .. 4096, any factors
static int check_line_bluestein(const char *who, int64_t n) {
    NBK_CHECK_ARG(n >= 2 && n <= NBK_MR_MAX_LINE,
                  "%s: line length %lld unsupported: the Bluestein FFT takes lengths 2 .. 4096", who, (long long)n);
    return NBK_OK;
}

static int check_z_bluestein(const char *who, int64_t Nz) {
    NBK_CHECK_ARG(Nz >= 2 && ((Nz % 2 == 0 && Nz <= 2 * NBK_MR_MAX_LINE) || (Nz % 2 && Nz < NBK_MR_MAX_LINE)),
                  "%s: Nz = %lld unsupported: the Bluestein z pass takes even lengths up to 8192 or odd lengths up to 4095",
                  who, (long long)Nz);
    return NBK_OK;
}

// shared bytes of one M-point tile of B lines, with or without W_M beside it
template <typename C>
static size_t bs_smem(int M, int B, bool tw_shared) {
    return ((size_t)M * (B > 1 ? B + 1 : 1) + (tw_shared ? M : 0)) * sizeof(C) + 16;
}

template <typename T>
static int launch_lines_bluestein(const void *src, void *dst, int N, int64_t line_stride, int64_t n_inner, int64_t n_outer,
                                  int64_t outer_stride, int inverse, double scale, cudaStream_t s) {
    typedef typename C2<T>::type C;
    const int dtype = sizeof(T) == 4 ? NBK_F4 : NBK_F8;
    const int M = bs_len(N);
    void *tw, *chirp, *filt;
    int rc = get_twiddle(M, dtype, s, &tw);
    if (rc) return rc;
    rc = get_bluestein(N, dtype, s, &chirp, &filt);
    if (rc) return rc;
    // 128-byte runs while two CTAs per SM fit, narrower for long lines
    int B = 128 / (int)sizeof(C);
    while (B > 1 && (bs_smem<C>(M, B, true) > 110 * 1024 || B / 2 >= n_inner)) B >>= 1;
    const int tw_shared = bs_smem<C>(M, B, true) <= 227 * 1024;
    const size_t smem = bs_smem<C>(M, B, tw_shared);
    NBK_CHECK_ARG(smem <= 227 * 1024, "fft_lines_bluestein: N=%d does not fit in shared memory", N);
    const int64_t tiles_inner = (n_inner + B - 1) / B;
    const int64_t n_tiles = tiles_inner * n_outer;
    int per_sm = (int)((227 * 1024) / (smem + 1024));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 8) per_sm = 8;
    const int64_t g = n_tiles < (int64_t)NBK_SM_COUNT * per_sm ? n_tiles : (int64_t)NBK_SM_COUNT * per_sm;
    const int nthreads = (per_sm == 1 && (int64_t)M * B >= 4096) ? 512 : 256;
    const MixedPlan plan = mr_plan(M);
#define LAUNCH_LB(BB)                                                                                                  \
    case BB:                                                                                                           \
        NBK_CUDA(cudaFuncSetAttribute(k_fft_lines_bluestein<T, BB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        k_fft_lines_bluestein<T, BB><<<(int)g, nthreads, smem, s>>>((const C *)src, (C *)dst, (const C *)tw, (const C *)chirp, \
                                                                     (const C *)filt, plan, N, line_stride, n_inner,      \
                                                                     tiles_inner, n_tiles, outer_stride, inverse, (T)scale, \
                                                                     tw_shared);                                          \
        break;
    switch (B) {
        LAUNCH_LB(1) LAUNCH_LB(2) LAUNCH_LB(4) LAUNCH_LB(8) LAUNCH_LB(16)
        default: nbk_set_error("fft_lines_bluestein: internal tile width %d", B); return NBK_ERR_ARG;
    }
#undef LAUNCH_LB
    NBK_LAUNCHED();
    return NBK_OK;
}

template <typename T>
static int launch_z_bluestein(const void *in, void *out, int64_t rows, int Nz, int inverse, double scale, cudaStream_t s) {
    typedef typename C2<T>::type C;
    const int dtype = sizeof(T) == 4 ? NBK_F4 : NBK_F8;
    const bool odd = Nz & 1;
    const int L = odd ? Nz : Nz / 2;
    const int M = bs_len(L);
    void *twz, *tw, *chirp, *filt;
    int rc = get_twiddle(Nz, dtype, s, &twz);
    if (rc) return rc;
    rc = get_twiddle(M, dtype, s, &tw);
    if (rc) return rc;
    rc = get_bluestein(L, dtype, s, &chirp, &filt);
    if (rc) return rc;
    const int64_t lines = odd ? (rows + 1) / 2 : rows;
    // B rows per tile: as many as leave two CTAs per SM; long rows take the whole SM
    int B = 16;
    while (B > 1 && (bs_smem<C>(M, B, true) > 110 * 1024 || B / 2 >= lines)) B >>= 1;
    const int tw_shared = bs_smem<C>(M, B, true) <= 227 * 1024;
    const size_t smem = bs_smem<C>(M, B, tw_shared);
    NBK_CHECK_ARG(smem <= 227 * 1024, "fft_z_bluestein: Nz=%d does not fit in shared memory", Nz);
    const int64_t n_tiles = (lines + B - 1) / B;
    int per_sm = (int)((227 * 1024) / (smem + 1024));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 8) per_sm = 8;
    const int64_t g = n_tiles < (int64_t)NBK_SM_COUNT * per_sm ? n_tiles : (int64_t)NBK_SM_COUNT * per_sm;
    const MixedPlan plan = mr_plan(M);
#define LAUNCH_ZB(BB)                                                                                                  \
    case BB:                                                                                                           \
        NBK_CUDA(cudaFuncSetAttribute(k_fft_z_bluestein<T, BB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        k_fft_z_bluestein<T, BB><<<(int)g, 256, smem, s>>>(in, out, (const C *)twz, (const C *)tw, (const C *)chirp,       \
                                                            (const C *)filt, plan, Nz, rows, inverse, (T)scale, tw_shared); \
        break;
    switch (B) {
        LAUNCH_ZB(1) LAUNCH_ZB(2) LAUNCH_ZB(4) LAUNCH_ZB(8) LAUNCH_ZB(16)
        default: nbk_set_error("fft_z_bluestein: internal tile width %d", B); return NBK_ERR_ARG;
    }
#undef LAUNCH_ZB
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_fft_lines_bluestein(const void *src, void *dst, int dtype, int64_t n_line, int64_t line_stride,
                                       int64_t n_inner, int64_t n_outer, int64_t outer_stride, int inverse, double scale,
                                       void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "fft_lines_bluestein: bad dtype %d", dtype);
    int rc = check_line_bluestein("fft_lines_bluestein", n_line);
    if (rc) return rc;
    if (n_inner <= 0 || n_outer <= 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == NBK_F4)
        return launch_lines_bluestein<float>(src, dst, (int)n_line, line_stride, n_inner, n_outer, outer_stride, inverse, scale, s);
    return launch_lines_bluestein<double>(src, dst, (int)n_line, line_stride, n_inner, n_outer, outer_stride, inverse, scale, s);
}

extern "C" int nbk_fft_z_bluestein(const void *in, void *out, int dtype, int64_t rows, int64_t Nz, int inverse, double scale,
                                   void *stream) {
    NBK_CHECK_ARG(dtype == NBK_F4 || dtype == NBK_F8, "fft_z_bluestein: bad dtype %d", dtype);
    int rc = check_z_bluestein("fft_z_bluestein", Nz);
    if (rc) return rc;
    if (rows <= 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    return (dtype == NBK_F4) ? launch_z_bluestein<float>(in, out, rows, (int)Nz, inverse, scale, s)
                             : launch_z_bluestein<double>(in, out, rows, (int)Nz, inverse, scale, s);
}
