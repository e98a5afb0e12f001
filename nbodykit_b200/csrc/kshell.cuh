// Fourier-slab geometry, the |k| bin of a mode and the Legendre weights of mu, shared by nbk_power_bin (binning.cu) and the bispectrum shells
// (bispectrum.cu), so that a shell of FFTBispectrum holds exactly the modes FFTPower puts in the same k bin.  Both
// translation units are built with --fmad=false: the float32 coordinate arithmetic that feeds k2 is part of that contract.
#pragma once
#include <math.h>
#include "common.cuh"

// ---------------------------------------------------------------------------------------------
// index helpers: element e of a slab -> integer frequency labels (jx, jy, jz)
// ---------------------------------------------------------------------------------------------
struct SlabGeom {
    int N[3];        // Nx, Ny, Nz of the full mesh
    int Nzc;         // stored length of the last axis
    int transposed;  // 0: [x_n][Ny][Nzc]   1: [y_n][Nx][Nzc]
    int start, count;  // owned range along the first stored axis
    int D1;          // length of the second stored axis
};

static int make_slab(const int64_t *nmesh, int transposed, int64_t start, int64_t count, int hermitian, SlabGeom &g) {
    for (int d = 0; d < 3; d++) {
        NBK_CHECK_ARG(nmesh[d] > 0 && nmesh[d] < (1 << 24), "bad Nmesh[%d]=%lld", d, (long long)nmesh[d]);
        g.N[d] = (int)nmesh[d];
    }
    // `transposed` carries the layout bits: NBK_LAYOUT_TRANSPOSED (first stored axis is y) and NBK_LAYOUT_FULLZ (the
    // last axis holds all Nz modes: complex-dtype meshes, real-space statistics)
    const bool fullz = (transposed & NBK_LAYOUT_FULLZ) != 0;
    transposed &= NBK_LAYOUT_TRANSPOSED;
    g.Nzc = (hermitian && !fullz) ? g.N[2] / 2 + 1 : g.N[2];
    g.transposed = transposed ? 1 : 0;
    int D0 = transposed ? g.N[1] : g.N[0];
    g.D1 = transposed ? g.N[0] : g.N[1];
    NBK_CHECK_ARG(start >= 0 && count >= 0 && start + count <= D0, "bad slab range [%lld,+%lld) of %d",
                  (long long)start, (long long)count, D0);
    g.start = (int)start;
    g.count = (int)count;
    return NBK_OK;
}

__device__ __forceinline__ void slab_freqs(const SlabGeom &g, int i0, int i1, int kz, int &jx, int &jy, int &jz) {
    int a = nbk_freq(g.start + i0, g.transposed ? g.N[1] : g.N[0]);
    int b = nbk_freq(i1, g.transposed ? g.N[0] : g.N[1]);
    jx = g.transposed ? b : a;
    jy = g.transposed ? a : b;
    jz = nbk_freq(kz, g.N[2]);
}

// number of edges <= x  (numpy.digitize, right=False, increasing edges)
__device__ __forceinline__ int digitize(const double *__restrict__ edges, int n, double x) {
    int lo = 0, hi = n;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (edges[mid] <= x) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// numpy.digitize(k2, k2edges) over nedge squared edges: 0 below the first edge, nedge at or above the last.  With
// uniform edges (numpy.arange: k2edges[i] = (kmin + i dk)^2 rounded), the bin starts from the closed-form guess
// (knorm - kmin) / dk and is corrected against the exact edges, so it equals the binary search for any increasing edges.
__device__ __forceinline__ int nbk_k2_bin(const double *__restrict__ k2edges, int nedge, double k2d, double knorm,
                                          double kmin, double inv_dk, int uniform) {
    if (!uniform) return digitize(k2edges, nedge, k2d);
    double t = (knorm - kmin) * inv_dk;
    int b = t < 0.0 ? 0 : (t >= (double)nedge ? nedge : (int)t + 1);
    while (b > 0 && k2d < k2edges[b - 1]) b--;
    while (b < nedge && k2d >= k2edges[b]) b++;
    return b;
}

// Legendre polynomial L_ell(x) in float64 by Bonnet's recurrence: the FFTPower multipole weights (nbk_power_bin) and
// the weights of the bispectrum multipole fields (nbk_bispec_fill_poles)
__device__ __forceinline__ double legendre(int ell, double x) {
    if (ell == 0) return 1.0;
    double p0 = 1.0, p1 = x;
    for (int n = 1; n < ell; n++) {
        double p2 = ((2 * n + 1) * x * p1 - n * p0) / (n + 1);
        p0 = p1;
        p1 = p2;
    }
    return p1;
}

// The last (x) pass of the forward transform fused with the FFTPower 1d auto-power binning (k_fft_x_bin in fft.cu,
// entry point nbk_fft_x_power_bin in binning.cu).  The mode's bin is the one nbk_power_bin gives it at float32
// coordinates with a line of sight along z and mu edges {-1, 1}; its accumulators are indexed key = kbin * 3 + mubin.
struct XBinArgs {
    int N[3], Nzc;
    float kf32[3], losz32;
    double volume;
    const double *k2edges;     // device, nedge = Nx + 1 squared edges
    int nedge;
    double kmin, inv_dk;
    int uniform;
    const double *ct0, *ct1, *ctz;   // per-axis reciprocal window factors (both fields), null without compensation
    unsigned long long *nsum;
    double *xsum, *ysum;       // ysum: (re, im) pairs
};
// *done = false: the shape does not take the fused kernel (line length, alignment, shared memory); nothing was launched
int fft_x_bin_launch(void *cplx, int dtype, double scale, const XBinArgs &a, cudaStream_t s, bool *done);

// host side of the uniform guess: are the nedge = Nx + 1 squared edges those of numpy.arange?  Sets kmin and 1/dk.
static inline int nbk_k2_uniform(const double *k2edges, int Nx, double *kmin, double *inv_dk) {
    *kmin = 0.0;
    *inv_dk = 0.0;
    int uniform = 0;
    if (Nx >= 1 && k2edges[0] >= 0.0) {
        *kmin = sqrt(k2edges[0]);
        double dk = (sqrt(k2edges[Nx]) - *kmin) / Nx;
        uniform = dk > 0.0;
        for (int i = 0; i <= Nx && uniform; i++)
            if (fabs(sqrt(k2edges[i]) - (*kmin + i * dk)) > 1e-3 * dk) uniform = 0;
        if (uniform) *inv_dk = 1.0 / dk;
    }
    return uniform;
}
