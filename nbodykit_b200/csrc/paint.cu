// Particle -> mesh window scatter (pmesh `pm.paint`, called from source/mesh/catalog.py:287,295-296).
//
// Compiled with --fmad=false: the grid coordinate g = fl(fl(double(pos)*fl(N/L)) + shift) and the
// f8 window weights must round exactly as the oracle does (SURVEY B.1/B.2); cell indices are
// bit-exact by contract.
//
// Path "direct": one particle per thread, support^3 native L2 reductions (REDG.E.ADD.F32/.F64)
// into the mesh.  sm_90a has no native shared-memory float/64-bit atomic add (ATOMS.CAST.SPIN
// loops), while REDG f32/f64 is native, so the mesh itself is the accumulator and the L2 (50 MB on H100) absorbs the
// read-modify-write of spatially coherent catalogues.
#include "common.cuh"
#include <stdlib.h>
#include <type_traits>

template <int SUP> struct Window;

// nearest grid point
template <> struct Window<1> {
    __device__ static __forceinline__ void eval(double g, long long &i0, double *w) {
        i0 = (long long)floor(g + 0.5);
        w[0] = 1.0;
    }
};
// CIC: i0 = floor(g), w = (1-d, d)
template <> struct Window<2> {
    __device__ static __forceinline__ void eval(double g, long long &i0, double *w) {
        double f = floor(g);
        double d = g - f;
        i0 = (long long)f;
        w[0] = 1.0 - d;
        w[1] = d;
    }
};
__device__ __forceinline__ double tsc_kernel(double x) {
    x = fabs(x);
    if (x <= 0.5) return 0.75 - x * x;
    if (x < 1.5) { double t = 1.5 - x; return 0.5 * (t * t); }
    return 0.0;
}
// TSC: i0 = floor(g + 0.5) - 1, w_r = K(g - i0 - r)
template <> struct Window<3> {
    __device__ static __forceinline__ void eval(double g, long long &i0, double *w) {
        double f = floor(g + 0.5) - 1.0;
        double d = g - f;
        i0 = (long long)f;
#pragma unroll
        for (int r = 0; r < 3; r++) w[r] = tsc_kernel(d - (double)r);
    }
};
__device__ __forceinline__ double pcs_kernel(double x) {
    x = fabs(x);
    if (x < 1.0) return (4.0 - 6.0 * x * x + 3.0 * (x * x * x)) / 6.0;
    if (x < 2.0) { double t = 2.0 - x; return (t * t * t) / 6.0; }
    return 0.0;
}
template <> struct Window<4> {
    __device__ static __forceinline__ void eval(double g, long long &i0, double *w) {
        double f = floor(g) - 1.0;
        double d = g - f;
        i0 = (long long)f;
#pragma unroll
        for (int r = 0; r < 4; r++) w[r] = pcs_kernel(d - (double)r);
    }
};

struct PaintGeom {
    double scale[3];   // fl(N_d / L_d)
    int n[3];          // Nmesh
    int x_start, x_n;  // owned x planes
};

__device__ __forceinline__ int wrap(long long i, int n) {
    // in-box particles (the overwhelming majority) never pay for the 64-bit modulo
    if ((unsigned long long)i < (unsigned long long)n) return (int)i;
    if (i >= -(long long)n && i < 2ll * n) return (int)(i < 0 ? i + n : i - n);
    long long r = i % n;
    return (int)(r < 0 ? r + n : r);
}

template <typename PT>
__device__ __forceinline__ bool load_grid(const PT *__restrict__ pos, int64_t i, const PaintGeom &gm,
                                          double shift, double *g) {
    bool ok = true;
#pragma unroll
    for (int d = 0; d < 3; d++) {
        double p = (double)pos[3 * i + d];
        g[d] = p * gm.scale[d] + shift;  // two roundings; this file is built with --fmad=false
        ok = ok && isfinite(g[d]);
    }
    return ok;
}

template <int SUP, typename FT>
__device__ __forceinline__ void scatter(const double *g, double mass, const PaintGeom &gm, FT *__restrict__ mesh) {
    long long i0[3];
    double w[3][SUP];
#pragma unroll
    for (int d = 0; d < 3; d++) Window<SUP>::eval(g[d], i0[d], w[d]);
    int iz[SUP], iy[SUP];
#pragma unroll
    for (int r = 0; r < SUP; r++) {
        iz[r] = wrap(i0[2] + r, gm.n[2]);
        iy[r] = wrap(i0[1] + r, gm.n[1]);
    }
#pragma unroll
    for (int rx = 0; rx < SUP; rx++) {
        int ix = wrap(i0[0] + rx, gm.n[0]) - gm.x_start;
        if (ix < 0 || ix >= gm.x_n) continue;  // ghost semantics: not my plane
#pragma unroll
        for (int ry = 0; ry < SUP; ry++) {
            double wxy = w[0][rx] * w[1][ry];
            int64_t row = ((int64_t)ix * gm.n[1] + iy[ry]) * gm.n[2];
#pragma unroll
            for (int rz = 0; rz < SUP; rz++) {
                double wt = wxy * w[2][rz] * mass;
                atomicAdd(&mesh[row + iz[rz]], (FT)wt);  // REDG.E.ADD.{F32,F64}
            }
        }
    }
}

template <int SUP, typename PT, typename MT, typename FT, bool INTERLACED>
__global__ void __launch_bounds__(256)
k_paint_direct(const PT *__restrict__ pos, const MT *__restrict__ mass, int64_t n, PaintGeom gm, double shift,
               FT *__restrict__ mesh, FT *__restrict__ mesh2) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        double g[3];
        double m = mass ? (double)mass[i] : 1.0;
        if (load_grid(pos, i, gm, shift, g)) scatter<SUP, FT>(g, m, gm, mesh);
        if (INTERLACED) {
            if (load_grid(pos, i, gm, 0.5, g)) scatter<SUP, FT>(g, m, gm, mesh2);
        }
    }
}

template <int SUP, typename PT>
__global__ void __launch_bounds__(256)
k_cell_index(const PT *__restrict__ pos, int64_t n, PaintGeom gm, double shift, int32_t *__restrict__ out) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        double g[3];
        bool ok = load_grid(pos, i, gm, shift, g);
#pragma unroll
        for (int d = 0; d < 3; d++) {
            long long i0 = 0;
            double w[SUP];
            if (ok) Window<SUP>::eval(g[d], i0, w);
            out[3 * i + d] = ok ? wrap(i0, gm.n[d]) : -1;
        }
    }
}

static int make_geom(const double *box, const int64_t *nmesh, int64_t x_start, int64_t x_n, PaintGeom &gm) {
    for (int d = 0; d < 3; d++) {
        NBK_CHECK_ARG(nmesh[d] > 0 && nmesh[d] < (1 << 30), "paint: bad Nmesh[%d]=%lld", d, (long long)nmesh[d]);
        NBK_CHECK_ARG(box[d] > 0, "paint: bad BoxSize[%d]=%g", d, box[d]);
        gm.n[d] = (int)nmesh[d];
        gm.scale[d] = (double)nmesh[d] / box[d];
    }
    NBK_CHECK_ARG(x_start >= 0 && x_n >= 0 && x_start + x_n <= nmesh[0], "paint: bad slab [%lld,+%lld)",
                  (long long)x_start, (long long)x_n);
    gm.x_start = (int)x_start;
    gm.x_n = (int)x_n;
    return NBK_OK;
}

template <int SUP, typename PT, typename MT, typename FT>
static int launch_paint2(const void *pos, const void *mass, int64_t n, const PaintGeom &gm, double shift, void *mesh,
                         void *mesh2, cudaStream_t s) {
    int g = nbk_grid_for(n, 256, 8);
    if (mesh2)
        k_paint_direct<SUP, PT, MT, FT, true>
            <<<g, 256, 0, s>>>((const PT *)pos, (const MT *)mass, n, gm, shift, (FT *)mesh, (FT *)mesh2);
    else
        k_paint_direct<SUP, PT, MT, FT, false>
            <<<g, 256, 0, s>>>((const PT *)pos, (const MT *)mass, n, gm, shift, (FT *)mesh, (FT *)nullptr);
    NBK_LAUNCHED();
    return NBK_OK;
}

template <int SUP, typename PT, typename MT>
static int launch_paint1(const void *pos, const void *mass, int64_t n, const PaintGeom &gm, double shift, void *mesh,
                         void *mesh2, int mesh_dtype, cudaStream_t s) {
    if (mesh_dtype == NBK_F4) return launch_paint2<SUP, PT, MT, float>(pos, mass, n, gm, shift, mesh, mesh2, s);
    return launch_paint2<SUP, PT, MT, double>(pos, mass, n, gm, shift, mesh, mesh2, s);
}

template <int SUP>
static int launch_paint0(const void *pos, int pos_dtype, const void *mass, int mass_dtype, int64_t n,
                         const PaintGeom &gm, double shift, void *mesh, void *mesh2, int mesh_dtype, cudaStream_t s) {
    bool pf4 = pos_dtype == NBK_F4, mf4 = (mass_dtype == NBK_F4);
    if (pf4 && mf4) return launch_paint1<SUP, float, float>(pos, mass, n, gm, shift, mesh, mesh2, mesh_dtype, s);
    if (pf4) return launch_paint1<SUP, float, double>(pos, mass, n, gm, shift, mesh, mesh2, mesh_dtype, s);
    if (mf4) return launch_paint1<SUP, double, float>(pos, mass, n, gm, shift, mesh, mesh2, mesh_dtype, s);
    return launch_paint1<SUP, double, double>(pos, mass, n, gm, shift, mesh, mesh2, mesh_dtype, s);
}

static int paint_impl(const void *pos, int pos_dtype, int64_t n, const void *mass, int mass_dtype, int window,
                      double shift, const double *box, const int64_t *nmesh, int64_t x_start, int64_t x_n,
                      void *mesh, void *mesh2, int mesh_dtype, void *stream) {
    NBK_CHECK_ARG(pos_dtype == NBK_F4 || pos_dtype == NBK_F8, "paint: bad pos dtype %d", pos_dtype);
    NBK_CHECK_ARG(mesh_dtype == NBK_F4 || mesh_dtype == NBK_F8, "paint: bad mesh dtype %d", mesh_dtype);
    NBK_CHECK_ARG(mass == nullptr || mass_dtype == NBK_F4 || mass_dtype == NBK_F8, "paint: bad mass dtype %d",
                  mass_dtype);
    NBK_CHECK_ARG(n >= 0, "paint: negative particle count");
    NBK_CHECK_ARG(mesh != nullptr, "paint: null mesh");
    PaintGeom gm;
    int rc = make_geom(box, nmesh, x_start, x_n, gm);
    if (rc) return rc;
    if (n == 0 || x_n == 0) return NBK_OK;
    if (mass == nullptr) mass_dtype = NBK_F8;
    cudaStream_t s = (cudaStream_t)stream;
    switch (window) {
        case NBK_WINDOW_NNB: return launch_paint0<1>(pos, pos_dtype, mass, mass_dtype, n, gm, shift, mesh, mesh2, mesh_dtype, s);
        case NBK_WINDOW_CIC: return launch_paint0<2>(pos, pos_dtype, mass, mass_dtype, n, gm, shift, mesh, mesh2, mesh_dtype, s);
        case NBK_WINDOW_TSC: return launch_paint0<3>(pos, pos_dtype, mass, mass_dtype, n, gm, shift, mesh, mesh2, mesh_dtype, s);
        case NBK_WINDOW_PCS: return launch_paint0<4>(pos, pos_dtype, mass, mass_dtype, n, gm, shift, mesh, mesh2, mesh_dtype, s);
    }
    nbk_set_error("paint: unknown window %d", window);
    return NBK_ERR_ARG;
}


// =============================================================================================
// Path "tiled": bucket particles by 16^3-cell tile, accumulate each tile in shared memory with
// native 32-bit integer atomics (ATOMS.ADD) on a 64-bit fixed-point representation, write every
// mesh cell exactly once.
//
// Shared u32 ATOMS in a CIC pattern sustain far more particles/s than the REDG path of "direct"
// (compare with tools/atomics_bench.cu), so the bucketing passes (HBM streaming) become the bound,
// independent of the particle order.  Fixed point also makes the mesh independent of the order particles arrive in:
// cell = round-to-nearest sum of w_i * 2^31/M, M = power of two >= max|mass| (exact integer
// adds, resolution 4.7e-10 M per deposit).
//
//   probe   k_bucket_probe    : samples neighbouring particle pairs: is the input spatially coherent (e.g. the
//                               cell-sorted output of a mock generator)?  Picks the bucketing configuration ON THE
//                               DEVICE (no host round trip): all configurations are launched, the others exit.
//                               Catalogues whose consecutive particles mostly share a tile take the RUN plan
//                               (k_run_count / k_run_place, see there): runs are bucketed instead of 12-byte records and
//                               the tile pass rebuilds each particle's record from its position.
//   pass A  k_bucket_count    : every CTA owns contiguous particle chunks (aligned quads per thread, 16-byte loads) and
//                               histograms the tile ids in a shared-memory WINDOW of tile indices (native
//                               ATOMS.ADD.U32); one global atomic per (chunk, tile) reserves the chunk's share of the
//                               tile's bucket.  Particles whose tile lies outside the window are counted with
//                               (warp-aggregated) global atomics.
//                               coherent input : window = 4 planes of tiles (<= 16384), 512-thread CTAs, 3 per SM
//                               scattered input: window = all tiles when they fit in 200 KB (<= 51200 tiles)
//   pass B  k_tile_scan(_totals): exclusive scan of the tile counts over segments of 4096 tiles -> bucket offsets;
//                               clears cursors and flags
//   pass C  k_bucket_scatter  : same chunks, same windows: evaluates the exact grid coordinate once and emits a
//                               12-byte record per particle (per axis: 4-bit cell-in-tile | 28-bit fraction); the
//                               records of a warp leave through a shared-memory transposition (coalesced stores)
//   pass D  k_tile_paint      : persistent CTAs pull tiles from a queue IN (descending) TILE ORDER; region = (T + halo)^3
//                               cells in shared memory as two u32 limbs.  Write-back without a cleared mesh and without
//                               read-modify-write of DRAM-resident lines: of all tiles touching a cell the FIRST in
//                               queue order stores it (plain coalesced stores) and publishes a per-tile flag
//                               (release); the later ones park their share and add it (REDG, L2-resident) one tile
//                               later if the earlier tiles have published -- otherwise they hand it to a deferred list
//                               (k_apply_deferred adds it after the kernel): nobody waits.  hold=True (accumulate into
//                               an existing mesh) uses one TMA bulk reduce-add per z row instead.
// A tile owns the particles whose LEFTMOST stencil cell lies in it, so the halo is one-sided.
// =============================================================================================
#define TILE 16
#define NBK_BLK_SMEM (200 * 1024)   // largest shared-memory tile window (scattered input)
#define NBK_WIN_COHERENT 16384      // tile window of the coherent configuration (64 KB)
#define NBK_CHUNKS_COHERENT (12 * NBK_SM_COUNT)
#define NBK_CHUNKS_SCATTERED NBK_SM_COUNT

// Tile-ordered particle record, 12 bytes for every position dtype: the scatter pass evaluates the grid coordinate
// in the exact f8 arithmetic once and stores, per axis, one word = leftmost stencil cell relative to its tile
// (high 4 bits) | fraction of (g + A) as 28-bit fixed point (truncated: the weights move by < 2^-28 = 3.7e-9).
// The paint pass needs no floor / wrap / range logic, and the half-cell shifted mesh of an interlaced pair follows
// exactly from frac + 1/2 (carry -> next cell).

struct TileGeom {
    PaintGeom gm;
    int G;            // ghost reach below the slab in x (0 when the slab is the whole mesh)
    int nt[3];        // tiles per axis
    int R;            // region edge = TILE + support - 1 (+1 when a half-cell shifted mesh is painted)
    int shifted;      // a half-cell shifted mesh is painted from the records (see shift_carry)
    int ntiles;
    int full;         // the slab is the whole mesh (single GPU): no ghost / ownership logic
};

// local x of a wrapped global cell relative to the slab origin, in [-G, Nx - G)
__device__ __forceinline__ int slab_local(int ix, const TileGeom &tg) {
    int lx = ix - tg.gm.x_start;
    if (lx >= tg.gm.n[0] - tg.G) lx -= tg.gm.n[0];
    if (lx < -tg.G) lx += tg.gm.n[0];
    return lx;
}

// leftmost-cell offsets of the windows: i0 = floor(g + OFF_A) + OFF_B
template <int SUP> struct WinOff;
template <> struct WinOff<1> { static constexpr float A = 0.5f; static constexpr int B = 0; };
template <> struct WinOff<2> { static constexpr float A = 0.0f; static constexpr int B = 0; };
template <> struct WinOff<3> { static constexpr float A = 0.5f; static constexpr int B = -1; };
template <> struct WinOff<4> { static constexpr float A = 0.0f; static constexpr int B = -1; };

__device__ __forceinline__ int tile_from_cells(const int *c, const TileGeom &tg) {
    if (tg.full)   // cells are in [0, n)
        return (int)((((unsigned)c[0] / TILE) * tg.nt[1] + (unsigned)c[1] / TILE) * tg.nt[2] + (unsigned)c[2] / TILE);
    int lx = slab_local(c[0], tg);
    if (lx < -tg.G || lx >= tg.gm.x_n) return -1;   // cannot touch my planes
    int tx = (lx + tg.G) / TILE, ty = c[1] / TILE, tz = c[2] / TILE;
    return (tx * tg.nt[1] + ty) * tg.nt[2] + tz;
}

// exact (f8) tile id of the particle at x[0..2]: the arithmetic of the scatter itself
// (coordinates by value: a pointer argument of a non-inlined function would force the callers' arrays into local memory)
template <int SUP, typename PT>
__device__ __noinline__ int tile_of_exact3(PT x0, PT x1, PT x2, const TileGeom &tg) {
    const PT x[3] = {x0, x1, x2};
    int c[3];
#pragma unroll
    for (int d = 0; d < 3; d++) {
        double g = (double)x[d] * tg.gm.scale[d];
        if (!isfinite(g)) return -1;
        long long i0;
        double w[SUP];
        Window<SUP>::eval(g, i0, w);
        c[d] = wrap(i0, tg.gm.n[d]);
    }
    return tile_from_cells(c, tg);
}
template <int SUP, typename PT>
__device__ __forceinline__ int tile_of_exact(const PT *x, const TileGeom &tg) { return tile_of_exact3<SUP, PT>(x[0], x[1], x[2], tg); }

__device__ __forceinline__ void pack_record(const unsigned *u, const int *c, const TileGeom &tg, unsigned *rec) {
    int lx = (tg.full ? c[0] : slab_local(c[0], tg) + tg.G) & (TILE - 1);
    rec[0] = (u[0] >> 4) | ((unsigned)lx << 28);
    rec[1] = (u[1] >> 4) | ((unsigned)(c[1] & (TILE - 1)) << 28);
    rec[2] = (u[2] >> 4) | ((unsigned)(c[2] & (TILE - 1)) << 28);
}

// The shifted mesh takes frac + 1/2 in fixed point, while the contract rounds in f8: g' = fl(a + 1/2) (po.grid_coords,
// the direct path).  Where fl(a + 1/2) rounds up onto the next integer (a + 1/2 below it by at most half an ulp: e.g.
// a = 1/2 - 2^-54) the contract's stencil starts one cell higher than the carry of the truncated fraction gives, and
// the shifted mesh would put a 2^-28 weight on a cell outside it.  There the record stores frac = 1/2 exactly, so the
// carry happens; the unshifted weights move by at most half an ulp of a + 1/2 (< 2^-28 for |g| < 2^24), within the
// truncation error the record already allows.
__device__ __forceinline__ unsigned shift_carry(unsigned u, double a, double f, const TileGeom &tg) {
    return (tg.shifted && u < 0x80000000u && (a + 0.5) - f >= 1.0) ? 0x80000000u : u;
}

// exact leftmost cell + fixed-point fraction (the arithmetic of Window<SUP>::eval on the unshifted g).
// Slow path: any magnitude, 64-bit cell arithmetic.
struct RecTile { unsigned r[3]; int tile; };
template <int SUP, typename PT>
__device__ __noinline__ RecTile make_record_slow3(PT x0, PT x1, PT x2, const TileGeom &tg) {
    const PT x[3] = {x0, x1, x2};
    RecTile o;
    o.r[0] = o.r[1] = o.r[2] = 0;
    o.tile = -1;
    unsigned u[3];
    int c[3];
#pragma unroll
    for (int d = 0; d < 3; d++) {
        double g = (double)x[d] * tg.gm.scale[d];
        if (!isfinite(g)) return o;
        double a = g + (double)WinOff<SUP>::A;
        double f = floor(a);
        u[d] = shift_carry(__double2uint_rz((a - f) * 4294967296.0), a, f, tg);
        c[d] = wrap((long long)f + WinOff<SUP>::B, tg.gm.n[d]);
    }
    pack_record(u, c, tg, o.r);
    o.tile = tile_from_cells(c, tg);
    return o;
}
template <int SUP, typename PT>
__device__ __forceinline__ int make_record_slow(const PT *x, const TileGeom &tg, unsigned *rec) {
    const RecTile o = make_record_slow3<SUP, PT>(x[0], x[1], x[2], tg);
    rec[0] = o.r[0]; rec[1] = o.r[1]; rec[2] = o.r[2];
    return o.tile;
}

// Fast path for |g| < 2^31 without any float<->int conversion instruction (they issue at a fraction of the FP64
// rate): a + 1.5*2^52 holds rint(a) in its low mantissa word; floor and the truncated 32-bit fraction follow with
// FP64 adds.  Bit-identical to the slow path.
template <int SUP, typename PT>
__device__ __forceinline__ int make_record(const PT *x, const TileGeom &tg, unsigned *rec) {
    const double K = 6755399441055744.0;      // 1.5 * 2^52
    unsigned u[3];
    int c[3];
    bool fast = true;
#pragma unroll
    for (int d = 0; d < 3; d++) {
        double a = (double)x[d] * tg.gm.scale[d];
        if (WinOff<SUP>::A != 0.f) a += (double)WinOff<SUP>::A;
        fast = fast && (fabs(a) < 2147483000.0);           // false for NaN / inf as well
        double r = a + K;
        int ri = __double2loint(r);
        double rf = r - K;                                  // rint(a)
        if (rf > a) { rf -= 1.0; ri -= 1; }                 // floor(a)
        // a - floor(a) rounds to 1.0 for a in (-2^-54, 0): saturate as the slow path's conversion does (2^32 would wrap
        // to a zero fraction and move the whole weight one cell down)
        const double fr = a - rf;
        u[d] = fr < 1.0 ? (unsigned)__double2loint(__dadd_rz(fr * 4294967296.0, 4503599627370496.0)) : 0xffffffffu;
        int cc = ri + WinOff<SUP>::B;                       // one period of wrap here, anything further in the slow path
        if (cc < 0) cc += tg.gm.n[d];
        else if (cc >= tg.gm.n[d]) cc -= tg.gm.n[d];
        fast = fast && ((unsigned)cc < (unsigned)tg.gm.n[d]);
        c[d] = cc;
    }
    // a half-cell shifted mesh takes the slow path, which applies shift_carry (the unshifted paints keep this path lean)
    if (!fast || tg.shifted) return make_record_slow<SUP, PT>(x, tg, rec);
    pack_record(u, c, tg, rec);
    return tile_from_cells(c, tg);      // the tile the bucketing pass counted this particle in (both are exact)
}

// per-launch constants of the float32 fast path of the tile id
struct FastTile {
    float sc[3];    // float32 scale N/L
    float lim[3];   // accept when |frac(g) - 0.5| < lim  (frac at least eps away from both cell boundaries)
    int pow2;       // N/L is a power of two on every axis: x * scale is exact in float32 (see make_record_pow2)
};

static FastTile make_fast_tile(const TileGeom &tg) {      // host side: passed to the kernels by value
    FastTile f;
    for (int d = 0; d < 3; d++) {
        f.sc[d] = (float)tg.gm.scale[d];
        // |g32 - g_exact| <= 2 float32 roundings of a value below n+2 -> 3e-7 (n+2) + 1e-6 is a safe margin
        f.lim[d] = 0.5f - (3e-7f * (float)(tg.gm.n[d] + 2) + 1e-6f);
    }
    f.pow2 = 1;
    for (int d = 0; d < 3; d++) {
        int e;
        if (frexp(tg.gm.scale[d], &e) != 0.5 || e < -60 || e > 60) f.pow2 = 0;
    }
    return f;
}

// float32 positions on a mesh whose N/L is a power of two (every benchmark box: L = 2 N): g = x * scale is EXACT in
// float32, so the leftmost cell and the 28-bit truncated fraction follow from float32 / integer arithmetic alone and
// are bit-identical to the f8 path (same real number, same truncation): ~8 instructions per axis instead of ~25.
// frac(g + 1/2) (TSC, NNB) is formed in fixed point: + 2^27 with the carry moving to the cell.  A float32 value plus 1/2
// is exact in f8, so the shifted mesh's carry already is the contract's rounding here (no shift_carry needed).
template <int SUP>
__device__ __forceinline__ int make_record_pow2(const float *x, const TileGeom &tg, const FastTile &ft, unsigned *rec, bool &ok) {
    unsigned u[3];
    int c[3];
    ok = true;
#pragma unroll
    for (int d = 0; d < 3; d++) {
        const float g = x[d] * ft.sc[d];                       // exact
        ok = ok && (fabsf(g) < 4194304.0f);                    // false for NaN / inf as well; far outside: slow path
        const float f = floorf(g);
        // (g - f) is exact except for g in (-2^-25, 0), where it rounds to 1.0: those take the f8 path, which rounds
        // g + A as the contract does
        const float fr = g - f;
        ok = ok && (fr < 1.0f);
        unsigned u28 = (unsigned)(fr * 268435456.0f);          // cvt truncates: floor(frac * 2^28)
        int ci = (int)f;
        if (WinOff<SUP>::A != 0.f) {
            u28 += 1u << 27;
            if (u28 >= (1u << 28)) { u28 -= 1u << 28; ci += 1; }
        }
        const int cc = ci + WinOff<SUP>::B;                  // a stencil that starts outside [0, n) wraps in the exact path
        ok = ok && ((unsigned)cc < (unsigned)tg.gm.n[d]);
        c[d] = cc;
        u[d] = u28 << 4;
    }
    if (!ok) return -1;
    pack_record(u, c, tg, rec);
    return tile_from_cells(c, tg);
}

// the record of one particle and its tile (-1: outside the slab): what the scatter pass stores and the run plan's
// tile pass rebuilds, bit for bit
template <int SUP, typename PT>
__device__ __forceinline__ int particle_record(const PT *x, const TileGeom &tg, const FastTile &ft, unsigned *rec) {
    bool okp = false;
    int t = -1;
    if (sizeof(PT) == 4 && ft.pow2) t = make_record_pow2<SUP>(reinterpret_cast<const float *>(x), tg, ft, rec, okp);
    if (!okp) t = make_record<SUP, PT>(x, tg, rec);
    return t;
}

// Tile id of a particle.  float32 in-box positions take a float32 fast path: unless the fraction of
// (x*scale + A) lies within the rounding margin of a cell boundary, floor() agrees with the exact f8 arithmetic;
// everything else (near-boundary, outside the box, f8 positions) is recomputed in f8 (ok == false).  The id is
// therefore ALWAYS the exact leftmost cell's tile -- count, scatter and paint passes agree.
template <int SUP, typename PT>
__device__ __forceinline__ int tile_fast(const PT *x, const TileGeom &tg, const FastTile &ft, bool &ok) {
    ok = sizeof(PT) == 4;
    int c[3] = {0, 0, 0};
    if (sizeof(PT) == 4 && ft.pow2) {
        // N/L a power of two: g = x * scale is exact in float32, so floor(g) IS the f8 result -- no margin test.  The
        // 1/2 of NNB / TSC is a carry on the exact fraction, as in make_record_pow2: g + 1/2 rounded in float32 is not
        // exact below 1/2 (g = 1/2 - 2^-25 gives 1.0), which put the count pass one cell -- for TSC one tile -- off
#pragma unroll
        for (int d = 0; d < 3; d++) {
            const float g = (float)x[d] * ft.sc[d];
            ok = ok && (fabsf(g) < 4194304.0f);                  // also false for NaN / inf
            int ci = __float2int_rd(g);
            if (WinOff<SUP>::A != 0.f && g - floorf(g) >= 0.5f) ci += 1;
            c[d] = ci + WinOff<SUP>::B;
            ok = ok && ((unsigned)c[d] < (unsigned)tg.gm.n[d]);
        }
    } else if (sizeof(PT) == 4) {
#pragma unroll
        for (int d = 0; d < 3; d++) {
            float g = (float)x[d] * ft.sc[d];
            if (WinOff<SUP>::A != 0.f) g += WinOff<SUP>::A;
            float f = floorf(g);
            ok = ok && (fabsf((g - f) - 0.5f) < ft.lim[d]);
            c[d] = (int)f + WinOff<SUP>::B;
            ok = ok && ((unsigned)c[d] < (unsigned)tg.gm.n[d]);
        }
    }
    return ok ? tile_from_cells(c, tg) : -1;
}

// one atomic per distinct key per warp; returns this lane's slot.  All 32 lanes must call.
__device__ __forceinline__ unsigned warp_claim(unsigned *counter, int key, bool active) {
    const int lane = threadIdx.x & 31;
    unsigned mask = __match_any_sync(0xffffffffu, active ? key : -1 - lane);
    if (!active) return 0;
    int leader = __ffs(mask) - 1;
    unsigned rank = __popc(mask & ((1u << lane) - 1));
    unsigned base = 0;
    if (lane == leader) base = atomicAdd(&counter[key], (unsigned)__popc(mask));
    base = __shfl_sync(mask, base, leader);
    return base + rank;
}

// Shared-memory counter claim.  Random catalogues: one native ATOMS per lane.  Spatially coherent catalogues put many
// lanes of a warp on the same counter, which the atomic unit serialises; when neighbouring lanes agree often, the
// warp aggregates equal keys first (one ATOMS per distinct key).  Must be called by all 32 lanes.
__device__ __forceinline__ unsigned smem_claim(unsigned *hist, int key, bool active) {
    const int lane = threadIdx.x & 31;
    int kn = __shfl_xor_sync(0xffffffffu, key, 1);
    unsigned same = __ballot_sync(0xffffffffu, active && kn == key);
    if (__popc(same) < 8) return active ? atomicAdd(&hist[key], 1u) : 0u;
    unsigned mask = __match_any_sync(0xffffffffu, active ? key : -1 - lane);
    if (!active) return 0u;
    int leader = __ffs(mask) - 1;
    unsigned base = 0;
    if (lane == leader) base = atomicAdd(&hist[key], (unsigned)__popc(mask));
    return __shfl_sync(mask, base, leader) + __popc(mask & ((1u << lane) - 1));
}

// Claim slots for the (up to) four particles of a thread's quad (k[u] = window-relative tile, -1 = none).
// Lanes run in array order, so for a spatially coherent catalogue the lanes whose whole quad lies in one tile form
// contiguous RUNS of equal keys: run heads come from one shuffle + ballot, the run's leader claims 4 * length slots
// with one native ATOMS and the members take consecutive groups of four (no MATCH.ANY).  The particles of quads that
// straddle tiles (and everything of a scattered catalogue) claim one slot each.  All 32 lanes must call.
__device__ __forceinline__ void quad_claim(unsigned *hist, const int (&k)[4], unsigned (&slot)[4]) {
    const unsigned lane = threadIdx.x & 31;
    const bool uni = (k[0] == k[1]) && (k[1] == k[2]) && (k[2] == k[3]) && (k[0] >= 0);
    const unsigned unis = __ballot_sync(0xffffffffu, uni);
    if (unis) {
        const int key = uni ? k[0] : -2 - (int)lane;                   // non-uniform lanes never join a run
        const int prev = __shfl_up_sync(0xffffffffu, key, 1);
        const unsigned heads = __ballot_sync(0xffffffffu, lane == 0 || prev != key);
        const unsigned below = heads & ((2u << lane) - 1u);            // heads at or below me (lane 31: all)
        const int start = 31 - __clz(lane == 31 ? heads : below);
        const unsigned above = lane == 31 ? 0u : (heads & ~((2u << lane) - 1u));
        const int end = above ? (__ffs(above) - 1) : 32;
        unsigned base = 0;
        if (uni && (int)lane == start) base = atomicAdd(&hist[key], 4u * (unsigned)(end - start));
        base = __shfl_sync(0xffffffffu, base, start);
        if (uni) {
            const unsigned s0 = base + 4u * (lane - (unsigned)start);
#pragma unroll
            for (int u = 0; u < 4; u++) slot[u] = s0 + u;
        }
    }
    if (!uni) {
#pragma unroll
        for (int u = 0; u < 4; u++) slot[u] = (k[u] >= 0) ? atomicAdd(&hist[k[u]], 1u) : 0u;
    }
}

// workspace header words
enum { HDR_QUEUE = 0, HDR_ABSMAX = 1, HDR_MODE = 2, HDR_DEFER = 3, HDR_WORDS = 64 };

struct BucketPlan {          // one bucketing configuration (host side, by value)
    int mode;                // value of the probe flag that selects this configuration
    int W;                   // tile window (entries of the shared histogram)
    int nchunks;             // particle chunks (CTAs loop over them)
    int64_t chunk;           // particles per chunk, multiple of 4
    int wstage;              // scatter pass: records leave through a per-warp shared-memory transposition (coalesced stores)
    int stage_off;           // ... byte offset of the warps' staging areas in dynamic shared memory
};

// Is the catalogue spatially coherent in array order?  256 threads sample neighbouring pairs (i, i+1): coherent pairs
// lie within one plane of tiles of each other.  mode <- 1 (coherent) when >= 3/4 of the valid pairs are.  The share of
// pairs in the SAME tile estimates 1 - 1 / (mean run length): mode <- 2 (runs) when it is >= 2/3, i.e. runs of >= 3
// particles on average, where bucketing runs moves fewer bytes than bucketing records (DESIGN.md 4.1).
template <int SUP, typename PT>
__global__ void __launch_bounds__(256)
k_bucket_probe(const PT *__restrict__ pos, int64_t n, TileGeom tg, int runs_ok, unsigned *__restrict__ hdr) {
    __shared__ int s_ok, s_tot, s_eq;
    if (threadIdx.x == 0) { s_ok = 0; s_tot = 0; s_eq = 0; }
    __syncthreads();
    const int plane = tg.nt[1] * tg.nt[2];
    int64_t j = (n > 1) ? (int64_t)((double)threadIdx.x / 256.0 * (double)(n - 1)) : 0;
    if (j + 1 < n) {
        PT a[3] = {pos[3 * j], pos[3 * j + 1], pos[3 * j + 2]};
        PT b[3] = {pos[3 * j + 3], pos[3 * j + 4], pos[3 * j + 5]};
        int ta = tile_of_exact<SUP, PT>(a, tg), tb = tile_of_exact<SUP, PT>(b, tg);
        if (ta >= 0 && tb >= 0) {
            atomicAdd(&s_tot, 1);
            int d = ta / plane - tb / plane;
            if (d >= -1 && d <= 1) atomicAdd(&s_ok, 1);
            if (ta == tb) atomicAdd(&s_eq, 1);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0)
        hdr[HDR_MODE] = (runs_ok && s_tot > 0 && 3 * s_eq >= 2 * s_tot) ? 2u : (s_tot > 0 && 4 * s_ok >= 3 * s_tot) ? 1u : 0u;
}

// quad of this thread, straight from global memory
template <typename PT>
__device__ __forceinline__ void load_quad_gmem(const PT *__restrict__ cpos, int j0, int nv, bool aligned, PT (&x)[4][3]) {
    if (aligned && nv == 4) {
        constexpr int NV = (int)(12 * sizeof(PT) / 16);
        const uint4 *v = reinterpret_cast<const uint4 *>(cpos + 3 * j0);
        uint4 r[NV];
#pragma unroll
        for (int k = 0; k < NV; k++) r[k] = v[k];
        const PT *f = reinterpret_cast<const PT *>(r);
#pragma unroll
        for (int u = 0; u < 4; u++) { x[u][0] = f[3 * u]; x[u][1] = f[3 * u + 1]; x[u][2] = f[3 * u + 2]; }
    } else {
#pragma unroll
        for (int u = 0; u < 4; u++) {
            bool in = u < nv;
            x[u][0] = in ? cpos[3 * (j0 + u)] : (PT)0;
            x[u][1] = in ? cpos[3 * (j0 + u) + 1] : (PT)0;
            x[u][2] = in ? cpos[3 * (j0 + u) + 2] : (PT)0;
        }
    }
}

__device__ __forceinline__ double load_mass(const void *mass, int mass_f4, int64_t i) {
    return mass_f4 ? (double)((const float *)mass)[i] : ((const double *)mass)[i];
}

// The chunk loop shared by the count and the scatter pass.  Rounds of 4 * blockDim particles: every thread owns one
// aligned quad per round.  `body(j0, nv, x)` is called by ALL threads (nv = 0 for idle ones) so that it may use warp
// collectives.
template <typename PT, typename F>
__device__ __forceinline__ void chunk_rounds(const PT *__restrict__ cpos, int cn, bool aligned, F body) {
    const int SP = 4 * (int)blockDim.x;                       // particles per round
    const int nround = (cn + SP - 1) / SP;
    for (int s = 0; s < nround; s++) {
        const int j0 = s * SP + 4 * (int)threadIdx.x;
        const int nv = min(4, max(0, cn - j0));
        PT x[4][3];
        load_quad_gmem(cpos, j0, nv, aligned, x);
        body(j0, nv, x);
    }
}

// exact tile ids of a quad (fast float32 path, exact recomputation where it is not decisive)
template <int SUP, typename PT>
__device__ __forceinline__ void quad_tiles(const PT (&x)[4][3], int nv, const TileGeom &tg, const FastTile &ft, int (&t)[4]) {
    bool redo = false;
    bool okv[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
        t[u] = tile_fast<SUP, PT>(x[u], tg, ft, okv[u]);
        redo = redo || (!okv[u] && u < nv);
    }
    if (redo) {                                  // rare: near a cell boundary / outside the box / f8 positions
#pragma unroll
        for (int u = 0; u < 4; u++)
            if (!okv[u] && u < nv) t[u] = tile_of_exact<SUP, PT>(x[u], tg);
    }
#pragma unroll
    for (int u = 0; u < 4; u++) if (u >= nv) t[u] = -1;
}

// window start of a chunk: 16 evenly spaced samples, the smallest plane of tiles among them minus one plane
template <int SUP, typename PT>
__device__ __forceinline__ int chunk_window_lo(const PT *__restrict__ cpos, int cn, const TileGeom &tg, int W, int *s_lo) {
    if (W >= tg.ntiles) return 0;
    if (threadIdx.x < 32) {
        int t = 0x7fffffff;
        if (threadIdx.x < 16 && cn > 0) {
            int j = (int)((int64_t)threadIdx.x * (cn - 1) / 15);
            PT x[3] = {cpos[3 * j], cpos[3 * j + 1], cpos[3 * j + 2]};
            int tt = tile_of_exact<SUP, PT>(x, tg);
            if (tt >= 0) t = tt;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t = min(t, __shfl_xor_sync(0xffffffffu, t, o));
        if (threadIdx.x == 0) {
            const int plane = tg.nt[1] * tg.nt[2];
            int lo = (t == 0x7fffffff) ? 0 : (t / plane - 1) * plane;
            lo = max(0, min(lo, tg.ntiles - W));
            *s_lo = lo;
        }
    }
    __syncthreads();
    return *s_lo;
}

// MAXT: 512 (coherent plan: three CTAs per SM -- the register cap that goes with it is what keeps the count pass at 40
// registers) or 1024 (scattered plan: one CTA per SM around a 200 KB histogram)
template <int SUP, typename PT, int MAXT>
__global__ void __launch_bounds__(MAXT, MAXT == 512 ? 3 : 1)
k_bucket_count(const PT *__restrict__ pos, const void *__restrict__ mass, int mass_f4, int64_t n, TileGeom tg, FastTile ft,
               unsigned *__restrict__ hdr, unsigned *__restrict__ cnt_w, unsigned *__restrict__ cnt_o,
               unsigned *__restrict__ blk, int *__restrict__ win_lo, BucketPlan bp) {
    if ((int)hdr[HDR_MODE] != bp.mode) return;
    extern __shared__ __align__(128) unsigned char s_raw[];
    unsigned *s_hist = reinterpret_cast<unsigned *>(s_raw);
    __shared__ int s_lo;
    const bool aligned = (reinterpret_cast<uintptr_t>(pos) & 15) == 0;
    float mx = 0.f;
    for (int c = blockIdx.x; c < bp.nchunks; c += gridDim.x) {
        const int64_t b = (int64_t)c * bp.chunk;
        const int64_t e = (b + bp.chunk < n) ? b + bp.chunk : n;
        const int cn = e > b ? (int)(e - b) : 0;
        const PT *cpos = pos + 3 * b;
        for (int i = threadIdx.x; i < bp.W; i += blockDim.x) s_hist[i] = 0;
        __syncthreads();
        const int lo = chunk_window_lo<SUP, PT>(cpos, cn, tg, bp.W, &s_lo);
        if (threadIdx.x == 0) win_lo[c] = lo;
        chunk_rounds<PT>(cpos, cn, aligned, [&](int j0, int nv, const PT (&x)[4][3]) {
            int t[4], k[4];
            quad_tiles<SUP, PT>(x, nv, tg, ft, t);
            bool anyout = false;
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const unsigned r = (unsigned)(t[u] - lo);
                k[u] = (t[u] >= 0 && r < (unsigned)bp.W) ? (int)r : -1;
                anyout = anyout || (t[u] >= 0 && k[u] < 0);
            }
            unsigned slot[4];
            quad_claim(s_hist, k, slot);
            if (__any_sync(0xffffffffu, anyout)) {
#pragma unroll
                for (int u = 0; u < 4; u++) warp_claim(cnt_o, t[u], t[u] >= 0 && k[u] < 0);
            }
            if (mass) {
#pragma unroll
                for (int u = 0; u < 4; u++)
                    if (t[u] >= 0) mx = fmaxf(mx, fabsf((float)load_mass(mass, mass_f4, b + j0 + u)) * 1.0000001f);
            }
        });
        __syncthreads();
        // reserve this chunk's share of every bucket: one global atomic per (chunk, tile)
        unsigned *row = blk + (size_t)c * bp.W;
        for (int i = threadIdx.x; i < bp.W; i += blockDim.x) {
            const unsigned h = s_hist[i];
            row[i] = h ? atomicAdd(&cnt_w[lo + i], h) : 0u;
        }
        __syncthreads();
    }
    if (mass) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if ((threadIdx.x & 31) == 0 && mx > 0.f) atomicMax(&hdr[HDR_ABSMAX], __float_as_uint(mx));  // positive floats order as uints
    }
}

// Exclusive scan of cnt_w + cnt_o -> bucket offsets, in two small launches over segments of 4096 tiles (a single CTA is
// a serial bottleneck for the 262 144 tiles of a 1024^3 mesh): (1) per-segment totals, (2) every segment adds the totals of the segments
// before it (<= 8192 of them: one strided pass of the CTA) to its local scan; also clears the outlier cursors, the per-tile
// flags and the tile queue head.
__global__ void __launch_bounds__(1024)
k_tile_scan_totals(const unsigned *__restrict__ cnt_w, const unsigned *__restrict__ cnt_o, unsigned *__restrict__ seg_tot, int ntiles) {
    __shared__ unsigned warp_tot[32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int i = blockIdx.x * 4096 + threadIdx.x * 4;
    unsigned s = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) if (i + j < ntiles) s += cnt_w[i + j] + cnt_o[i + j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) warp_tot[wid] = s;
    __syncthreads();
    if (wid == 0) {
        unsigned x = warp_tot[lane];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
        if (lane == 0) seg_tot[blockIdx.x] = x;
    }
}

__global__ void __launch_bounds__(1024)
k_tile_scan(const unsigned *__restrict__ cnt_w, const unsigned *__restrict__ cnt_o, const unsigned *__restrict__ seg_tot,
            unsigned *__restrict__ offsets, unsigned *__restrict__ cur_o, unsigned *__restrict__ flags, unsigned *__restrict__ hdr,
            int ntiles) {
    __shared__ unsigned warp_tot[32];
    __shared__ unsigned s_carry;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    // totals of the segments before mine (and, in the last segment, of all of them)
    unsigned before = 0;
    for (int b = threadIdx.x; b < (int)blockIdx.x; b += blockDim.x) before += seg_tot[b];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) before += __shfl_xor_sync(0xffffffffu, before, o);
    if (lane == 0) warp_tot[wid] = before;
    __syncthreads();
    if (wid == 0) {
        unsigned x = warp_tot[lane];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
        if (lane == 0) s_carry = x;
    }
    __syncthreads();
    const unsigned carry = s_carry;
    __syncthreads();
    const int i = blockIdx.x * 4096 + threadIdx.x * 4;
    unsigned v[4];
#pragma unroll
    for (int j = 0; j < 4; j++) v[j] = (i + j < ntiles) ? cnt_w[i + j] + cnt_o[i + j] : 0u;
    const unsigned s = v[0] + v[1] + v[2] + v[3];
    unsigned inc = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        unsigned nn = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += nn;
    }
    if (lane == 31) warp_tot[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        unsigned x = warp_tot[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            unsigned nn = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += nn;
        }
        warp_tot[lane] = x;
    }
    __syncthreads();
    unsigned run = carry + (wid ? warp_tot[wid - 1] : 0u) + inc - s;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        if (i + j < ntiles) { offsets[i + j] = run; cur_o[i + j] = 0; flags[i + j] = 0; }
        run += v[j];
    }
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) { offsets[ntiles] = carry + warp_tot[31]; hdr[HDR_QUEUE] = 0; }
}

template <int SUP, typename PT, int MAXT>
__global__ void __launch_bounds__(MAXT, MAXT == 512 ? 2 : 1)
k_bucket_scatter(const PT *__restrict__ pos, const void *__restrict__ mass, int mass_f4, int64_t n, TileGeom tg, FastTile ft,
                 const unsigned *__restrict__ hdr, const unsigned *__restrict__ offsets,
                 const unsigned *__restrict__ cnt_w, unsigned *__restrict__ cur_o, const unsigned *__restrict__ blk,
                 const int *__restrict__ win_lo, unsigned *__restrict__ recs, void *__restrict__ smass, BucketPlan bp) {
    if ((int)hdr[HDR_MODE] != bp.mode) return;
    extern __shared__ __align__(128) unsigned char s_raw[];
    unsigned *s_cur = reinterpret_cast<unsigned *>(s_raw);
    const bool aligned = (reinterpret_cast<uintptr_t>(pos) & 15) == 0;
    for (int c = blockIdx.x; c < bp.nchunks; c += gridDim.x) {
        const int64_t b = (int64_t)c * bp.chunk;
        const int64_t e = (b + bp.chunk < n) ? b + bp.chunk : n;
        const int cn = e > b ? (int)(e - b) : 0;
        const PT *cpos = pos + 3 * b;
        const int lo = win_lo[c];
        const unsigned *row = blk + (size_t)c * bp.W;
        const int wn = min(bp.W, tg.ntiles - lo);
        for (int i = threadIdx.x; i < wn; i += blockDim.x) s_cur[i] = offsets[lo + i] + row[i];
        __syncthreads();
        chunk_rounds<PT>(cpos, cn, aligned, [&](int j0, int nv, const PT (&x)[4][3]) {
            unsigned r[4][3];
            int t[4], k[4];
            bool anyout = false;
#pragma unroll
            for (int u = 0; u < 4; u++) {
                r[u][0] = r[u][1] = r[u][2] = 0;
                t[u] = -1;
                if (u < nv) t[u] = particle_record<SUP, PT>(x[u], tg, ft, r[u]);
                const unsigned rel = (unsigned)(t[u] - lo);
                k[u] = (t[u] >= 0 && rel < (unsigned)bp.W) ? (int)rel : -1;
                anyout = anyout || (t[u] >= 0 && k[u] < 0);
            }
            unsigned slot[4];
            quad_claim(s_cur, k, slot);
            if (__any_sync(0xffffffffu, anyout)) {
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const bool out = t[u] >= 0 && k[u] < 0;
                    unsigned so = warp_claim(cur_o, t[u], out);
                    if (out) slot[u] = offsets[t[u]] + cnt_w[t[u]] + so;     // outliers follow the windowed shares
                }
            }
            if (bp.wstage) {
                // Coalesced record stores.  A lane's quad is 12 words at 4 (mostly consecutive) slots: written straight
                // from the registers, every STG of the warp touches ~30 sectors (4 bytes each, 48 bytes apart) and the L1
                // store path -- not DRAM -- bounds the pass.  Instead the warp parks its 128 records (+ their word
                // offsets) in shared memory and writes them back with consecutive lanes on consecutive records.  (Word-by-
                // word order -- 128 contiguous bytes per STG -- needs a division by 3 per word and measured issue-bound.)
                unsigned *st = reinterpret_cast<unsigned *>(s_raw + bp.stage_off) + (threadIdx.x >> 5) * 512;
                const int lane = threadIdx.x & 31;
                // three word planes [k][record] + the records' word offsets 3 * slot (0xffffffff: no record)
#pragma unroll
                for (int k = 0; k < 3; k++)
                    reinterpret_cast<uint4 *>(st + 128 * k)[lane] = make_uint4(r[0][k], r[1][k], r[2][k], r[3][k]);
                reinterpret_cast<uint4 *>(st + 384)[lane] = make_uint4(t[0] >= 0 ? 3u * slot[0] : 0xffffffffu, t[1] >= 0 ? 3u * slot[1] : 0xffffffffu,
                                                                        t[2] >= 0 ? 3u * slot[2] : 0xffffffffu, t[3] >= 0 ? 3u * slot[3] : 0xffffffffu);
                __syncwarp();
                // lane <-> record rid = 32 jj + lane: consecutive lanes hold consecutive slots inside a run of equal tiles,
                // so a warp store covers a 384-byte span (12 sectors) instead of 32 scattered sectors
#pragma unroll
                for (int jj = 0; jj < 4; jj++) {
                    const int rid = jj * 32 + lane;
                    const unsigned o3 = st[384 + rid];
                    if (o3 != 0xffffffffu) {
                        unsigned *dst = recs + (size_t)o3;
                        dst[0] = st[rid]; dst[1] = st[128 + rid]; dst[2] = st[256 + rid];
                    }
                }
                __syncwarp();                                  // the next round overwrites the staging area
            }
#pragma unroll
            for (int u = 0; u < 4; u++) {
                if (t[u] >= 0) {
                    // 12-byte records (a 16-byte record, one vector store / load, makes the tile pass 25 % slower: it is
                    // the DRAM bytes that count)
                    if (!bp.wstage) {
                        unsigned *dst = recs + 3 * (size_t)slot[u];
                        dst[0] = r[u][0]; dst[1] = r[u][1]; dst[2] = r[u][2];
                    }
                    if (mass) {
                        if (mass_f4) ((float *)smass)[slot[u]] = ((const float *)mass)[b + j0 + u];
                        else ((double *)smass)[slot[u]] = ((const double *)mass)[b + j0 + u];
                    }
                }
            }
        });
        __syncthreads();
    }
}

// ---- run plan (mode 2).  A RUN is a maximal stretch of consecutive particles with the same tile inside one warp's
// 128-particle slice of a round.  Entry = {first particle, tile << 7 | (length - 1)}; the runs of chunk c fill the
// chunk's own region [c * chunk, ...) of the run list, so the list (one entry per particle at most) cannot overflow.
#define RUN_TILE_BITS 25

// pass A of the run plan: the count pass's chunks, window and exact tile ids, but one histogram count per RUN; writes
// the runs and their number per chunk
template <int SUP, typename PT>
__global__ void __launch_bounds__(512, 2)
k_run_count(const PT *__restrict__ pos, const void *__restrict__ mass, int mass_f4, int64_t n, TileGeom tg, FastTile ft,
            unsigned *__restrict__ hdr, unsigned *__restrict__ cnt_w, unsigned *__restrict__ cnt_o,
            unsigned *__restrict__ blk, int *__restrict__ win_lo, uint2 *__restrict__ runs, unsigned *__restrict__ run_n,
            BucketPlan bp) {
    if ((int)hdr[HDR_MODE] != bp.mode) return;
    extern __shared__ __align__(128) unsigned char s_raw[];
    unsigned *s_hist = reinterpret_cast<unsigned *>(s_raw);
    __shared__ int s_lo;
    __shared__ unsigned s_nrun;
    const bool aligned = (reinterpret_cast<uintptr_t>(pos) & 15) == 0;
    const unsigned lane = threadIdx.x & 31;
    float mx = 0.f;
    for (int c = blockIdx.x; c < bp.nchunks; c += gridDim.x) {
        const int64_t b = (int64_t)c * bp.chunk;
        const int64_t e = (b + bp.chunk < n) ? b + bp.chunk : n;
        const int cn = e > b ? (int)(e - b) : 0;
        const PT *cpos = pos + 3 * b;
        uint2 *crun = runs + b;
        for (int i = threadIdx.x; i < bp.W; i += blockDim.x) s_hist[i] = 0;
        if (threadIdx.x == 0) s_nrun = 0;
        __syncthreads();
        const int lo = chunk_window_lo<SUP, PT>(cpos, cn, tg, bp.W, &s_lo);
        if (threadIdx.x == 0) win_lo[c] = lo;
        chunk_rounds<PT>(cpos, cn, aligned, [&](int j0, int nv, const PT (&x)[4][3]) {
            int t[4];
            quad_tiles<SUP, PT>(x, nv, tg, ft, t);
            // boundaries: the slice's first particle and every tile change (t = -1 ends a run and starts none)
            const int prev = __shfl_up_sync(0xffffffffu, t[3], 1);
            bool bnd[4];
            bnd[0] = lane == 0 || prev != t[0];
#pragma unroll
            for (int u = 1; u < 4; u++) bnd[u] = t[u] != t[u - 1];
            unsigned B[4], H[4];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                B[u] = __ballot_sync(0xffffffffu, bnd[u]);
                H[u] = __ballot_sync(0xffffffffu, bnd[u] && t[u] >= 0);
            }
            // first boundary after this lane's quad (slice position 4 * lane + u), 128 = end of the slice
            const unsigned above = (B[0] | B[1] | B[2] | B[3]) & ~((2u << lane) - 1u);
            int next = 128;
            if (above) {
                const int L = __ffs(above) - 1;
                next = 4 * L + (((B[0] >> L) & 1u) ? 0 : ((B[1] >> L) & 1u) ? 1 : ((B[2] >> L) & 1u) ? 2 : 3);
            }
            int len[4];
#pragma unroll
            for (int u = 3; u >= 0; u--) {
                const int p = 4 * (int)lane + u;
                len[u] = next - p;
                if (bnd[u]) next = p;
            }
            const unsigned lt = (1u << lane) - 1u;
            unsigned rank = 0, tot = 0;
#pragma unroll
            for (int u = 0; u < 4; u++) { rank += __popc(H[u] & lt); tot += __popc(H[u]); }
            unsigned base = 0;
            if (lane == 0 && tot) base = atomicAdd(&s_nrun, tot);
            rank += __shfl_sync(0xffffffffu, base, 0);
            bool anyout = false;
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const bool head = (H[u] >> lane) & 1u;
                const unsigned r = (unsigned)(t[u] - lo);
                if (head) {
                    if (r < (unsigned)bp.W) atomicAdd(&s_hist[r], 1u);
                    else anyout = true;
                    crun[rank++] = make_uint2((unsigned)(b + j0 + u), ((unsigned)t[u] << 7) | (unsigned)(len[u] - 1));
                }
            }
            if (__any_sync(0xffffffffu, anyout)) {
#pragma unroll
                for (int u = 0; u < 4; u++)
                    warp_claim(cnt_o, t[u], ((H[u] >> lane) & 1u) && (unsigned)(t[u] - lo) >= (unsigned)bp.W);
            }
            if (mass) {
#pragma unroll
                for (int u = 0; u < 4; u++)
                    if (t[u] >= 0) mx = fmaxf(mx, fabsf((float)load_mass(mass, mass_f4, b + j0 + u)) * 1.0000001f);
            }
        });
        __syncthreads();
        unsigned *row = blk + (size_t)c * bp.W;
        for (int i = threadIdx.x; i < bp.W; i += blockDim.x) {
            const unsigned h = s_hist[i];
            row[i] = h ? atomicAdd(&cnt_w[lo + i], h) : 0u;
        }
        if (threadIdx.x == 0) run_n[c] = s_nrun;
        __syncthreads();
    }
    if (mass) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if ((threadIdx.x & 31) == 0 && mx > 0.f) atomicMax(&hdr[HDR_ABSMAX], __float_as_uint(mx));
    }
}

// pass C of the run plan: reads no positions; claims one bucket slot per run of the chunk (as k_bucket_scatter claims
// one per particle) and stores the run's index in the run list there
__global__ void __launch_bounds__(512)
k_run_place(const uint2 *__restrict__ runs, const unsigned *__restrict__ run_n, int ntiles, const unsigned *__restrict__ hdr,
            const unsigned *__restrict__ offsets, const unsigned *__restrict__ cnt_w, unsigned *__restrict__ cur_o,
            const unsigned *__restrict__ blk, const int *__restrict__ win_lo, unsigned *__restrict__ bucket, BucketPlan bp) {
    if ((int)hdr[HDR_MODE] != bp.mode) return;
    extern __shared__ __align__(128) unsigned char s_raw[];
    unsigned *s_cur = reinterpret_cast<unsigned *>(s_raw);
    for (int c = blockIdx.x; c < bp.nchunks; c += gridDim.x) {
        const int lo = win_lo[c];
        const unsigned *row = blk + (size_t)c * bp.W;
        const int wn = min(bp.W, ntiles - lo);
        for (int i = threadIdx.x; i < wn; i += blockDim.x) s_cur[i] = offsets[lo + i] + row[i];
        __syncthreads();
        const unsigned nr = run_n[c];
        const unsigned r0 = (unsigned)((int64_t)c * bp.chunk);
        for (unsigned i0 = 0; i0 < nr; i0 += blockDim.x) {
            const unsigned i = i0 + threadIdx.x;
            const bool valid = i < nr;
            const int t = valid ? (int)(runs[r0 + i].y >> 7) : -1;
            const unsigned k = (unsigned)(t - lo);
            const bool out = valid && k >= (unsigned)bp.W;
            unsigned slot = (valid && !out) ? atomicAdd(&s_cur[k], 1u) : 0u;
            if (__any_sync(0xffffffffu, out)) {
                const unsigned so = warp_claim(cur_o, t, out);
                if (out) slot = offsets[t] + cnt_w[t] + so;
            }
            if (valid) bucket[slot] = r0 + i;
        }
        __syncthreads();
    }
}

// 64-bit fixed-point cell = two 32-bit limbs kept in SEPARATE arrays lo[NC] | hi[NC] (so the low-limb atomics, which
// are nearly all of them, spread over all 32 banks).  Deposits are native ATOMS.ADD on the low limb; the carry (seen
// in the returned old value) goes to the high limb.
__device__ __forceinline__ void fixed_add(unsigned *lo, unsigned *hi, int cell, long long q) {
    unsigned ql = (unsigned)q, qh = (unsigned)(q >> 32);
    unsigned old = atomicAdd(&lo[cell], ql);
    unsigned h = qh + (unsigned)(old + ql < old);
    if (h) atomicAdd(&hi[cell], h);
}
// non-negative deposit: 0 <= q <= 2^31 fits the low limb
__device__ __forceinline__ void fixed_add_pos(unsigned *lo, unsigned *hi, int cell, unsigned ql) {
    unsigned old = atomicAdd(&lo[cell], ql);
    if (old + ql < old) atomicAdd(&hi[cell], 1u);
}

__device__ __forceinline__ void tma_reduce_add(double *gdst, const void *ssrc, unsigned bytes) {
    unsigned sa = (unsigned)__cvta_generic_to_shared(ssrc);
    asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f64 [%0], [%1], %2;"
                 :: "l"(gdst), "r"(sa), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_reduce_add(float *gdst, const void *ssrc, unsigned bytes) {
    unsigned sa = (unsigned)__cvta_generic_to_shared(ssrc);
    asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;"
                 :: "l"(gdst), "r"(sa), "r"(bytes) : "memory");
}

// window weights from the stencil-relative offset d = g - i0 (d in [0,1) CIC, [0.5,1.5) TSC, [1,2) PCS)
template <int SUP> struct WinD;
template <> struct WinD<1> { static constexpr double DMIN = 0.0;
    __device__ static __forceinline__ void eval(double, double *w) { w[0] = 1.0; } };
template <> struct WinD<2> { static constexpr double DMIN = 0.0;
    __device__ static __forceinline__ void eval(double d, double *w) { w[0] = 1.0 - d; w[1] = d; } };
template <> struct WinD<3> { static constexpr double DMIN = 0.5;
    __device__ static __forceinline__ void eval(double d, double *w) {
#pragma unroll
        for (int r = 0; r < 3; r++) w[r] = tsc_kernel(d - (double)r);
    } };
template <> struct WinD<4> { static constexpr double DMIN = 1.0;
    __device__ static __forceinline__ void eval(double d, double *w) {
#pragma unroll
        for (int r = 0; r < 4; r++) w[r] = pcs_kernel(d - (double)r);
    } };

__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
// polling load: gpu-scope relaxed (no L1 invalidation per iteration, unlike ld.acquire = LDG.STRONG + CCTL.IVALL);
// the acquire is one fence after the loop
__device__ __forceinline__ unsigned ld_relaxed(const unsigned *p) {
    unsigned v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void fence_acq_rel_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
__device__ __forceinline__ void st_release(unsigned *p, unsigned v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}

// Along every axis a region cell with local coordinate a is touched by this tile, by the preceding tile if a < H and
// by the following one if a >= TILE.  Tiles are handed out in DESCENDING index order (lexicographic in (tx, ty, tz)),
// so along each axis the tile with the larger coordinate is the earlier one and the first toucher of a cell is the
// per-axis maximum: an interior tile is first for exactly its own 16^3 base block (rows of 16 cells = aligned
// 128-byte runs of an f8 mesh) and adds its halo to the blocks of the tiles that came before it.  [flo, fhi) = the
// local coordinates this tile is first for along the axis; the periodic seam is the exception: tile 0's predecessor
// is the LAST tile (earlier), and the last tile's successor is tile 0 (later).
struct TileBox {
    int tc[3], o[3], flo[3], fhi[3];
};
template <int R, int H>
__device__ __forceinline__ TileBox tile_box(int t, const TileGeom &tg) {
    TileBox b;
    b.tc[2] = t % tg.nt[2];
    b.tc[1] = (t / tg.nt[2]) % tg.nt[1];
    b.tc[0] = t / (tg.nt[2] * tg.nt[1]);
    b.o[0] = b.tc[0] * TILE - tg.G;                  // region origin (x: slab-local)
    b.o[1] = b.tc[1] * TILE;
    b.o[2] = b.tc[2] * TILE;
#pragma unroll
    for (int d = 0; d < 3; d++) {
        const bool periodic = (d > 0) || tg.full;
        b.flo[d] = (periodic && b.tc[d] == 0) ? H : 0;
        b.fhi[d] = (b.tc[d] < tg.nt[d] - 1) ? TILE : R;
    }
    return b;
}

// exact (double)(hi:lo as a signed 64-bit integer) without conversion instructions (2^52 mantissa trick, one rounding)
__device__ __forceinline__ double limbs_to_double(unsigned lo, unsigned hi) {
    const double dlo = __hiloint2double(0x43300000, (int)lo) - 4503599627370496.0;
    const double dhi = __hiloint2double(0x43300000, (int)(hi ^ 0x80000000u)) - 4503601774854144.0;   // 2^52 + 2^31
    return __fma_rn(dhi, 4294967296.0, dlo);
}

template <bool V> struct BoolTag { static constexpr bool value = V; };

__host__ __device__ constexpr int tile_plane_pitch(int sup, int flush, int R, int RP) {
    int ps = R * RP;
    if (sup == 2 && flush == 0) ps += (8 - (ps & 31) + 32) & 31;     // even: R * RP and 8 are
    return ps;
}

// FLUSH 0: ordered write-back: of all tiles touching a cell the first in queue order stores it (plain coalesced
//          stores), the later ones add (REDG, L2-resident) after the earlier tiles have published their stores; no
//          cleared mesh needed, every cell is written exactly once.  Interior tiles (the common case) store their own
//          16^3 base block as 16-byte pairs straight from the accumulator and park their halo -- the cells they must
//          ADD to the blocks of earlier tiles -- in a small shared-memory stash, which is added one tile later, after
//          the CTA has accumulated its next tile: by then the neighbours have long published, so the flag poll (per
//          warp, no CTA barrier) is almost never a wait.  Two CTA barriers per tile.  Tiles on the mesh boundary take
//          a generic per-cell path (and wait in place where their add set does not fit the stash).
// FLUSH 1: TMA bulk reduce-add, one row per op, into an existing mesh (hold=True)
// PT void: the record plans -- recs = 12-byte records, smass = their masses in bucket order.  PT float / double: the run
// plan -- recs = run indices, runs = the run list, pos and smass = the catalogue's positions and masses; the records are
// rebuilt from the positions (particle_record, bit for bit the scatter pass's), so the mesh is the record plans' mesh.
template <int SUP, typename MT, typename FT, bool SHIFTED, int FLUSH, typename PT>
__global__ void __launch_bounds__(256, FLUSH == 0 ? 4 : 1)
k_tile_paint(const unsigned *__restrict__ recs, const MT *__restrict__ smass, TileGeom tg,
             const unsigned *__restrict__ offsets, unsigned *__restrict__ hdr, unsigned *__restrict__ flags,
             unsigned epoch, FT *__restrict__ mesh, unsigned *__restrict__ d_off, FT *__restrict__ d_val, unsigned d_cap,
             const uint2 *__restrict__ runs, const PT *__restrict__ pos, FastTile ft) {
    constexpr bool RUNS = !std::is_void<PT>::value;
    if ((hdr[HDR_MODE] == 2u) != RUNS) return;
    extern __shared__ __align__(16) unsigned s_all[];
    constexpr int R = TILE + SUP - 1 + (SHIFTED ? 1 : 0);   // == tg.R
    // row pitch in cells: the TMA write-back needs rows that start 16-byte aligned, the ordered one 8-byte cell pairs
    constexpr int RP = FLUSH == 0 ? ((R + 1) & ~1) : ((R + 3) & ~3);
    // x-plane pitch.  CIC, ordered write-back: padded so that the 8 corners of a stencil fall into 8 different banks
    // (offsets {0, 1, RP, RP+1} + {0, PS}: PS = 8 mod 32 with RP = 18); the padding measurably changes the speed
    constexpr int PS = tile_plane_pitch(SUP, FLUSH, R, RP);
    constexpr int NC = R * PS;
    constexpr int BUFW = (2 * NC + 3) & ~3;                  // words of the accumulator (lo | hi limbs)
    constexpr int H = R - TILE;   // cells with a local coordinate < H are also written by the preceding tile
    constexpr int CAP = R * R * R - TILE * TILE * TILE;      // halo cells = what an interior tile adds
    constexpr int NT = 256;
    constexpr int HK = (CAP + NT - 1) / NT;                  // halo cells per thread
    unsigned *s_lo = s_all, *s_hi = s_all + NC;
    FT *s_sval = reinterpret_cast<FT *>(s_all + BUFW);                    // stash: value ...
    unsigned *s_soff = reinterpret_cast<unsigned *>(s_sval + CAP);        // ... and mesh offset of a parked cell
    __shared__ int s_tile;
    __shared__ unsigned s_nst[2];
    // scale 2^31 / M, M = power of two >= max |mass|
    double M = 1.0;
    if (smass) {
        float mx = __uint_as_float(hdr[HDR_ABSMAX]);
        int e;
        frexpf(mx, &e);
        M = mx > 0.f ? ldexp(1.0, e) : 1.0;
    }
    const double S = 2147483648.0 / M, invS = M / 2147483648.0;
    for (int i = threadIdx.x; i < BUFW / 4; i += NT) reinterpret_cast<uint4 *>(s_all)[i] = make_uint4(0, 0, 0, 0);
    if (threadIdx.x == 0) { s_nst[0] = 0; s_nst[1] = 0; }
    const bool small_mesh = (int64_t)tg.gm.x_n * tg.gm.n[1] * tg.gm.n[2] < (1ll << 32);   // 32-bit stash offsets
    const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const unsigned sbase = smem_u32(s_lo);
    constexpr unsigned HIOFF = 4u * (unsigned)NC;          // low limb -> high limb, bytes
    // non-negative deposit q <= 2^31 at the low limb `addr` (shared-window byte address); the carry goes to the high limb
    auto deposit = [&](unsigned addr, unsigned q) {
        // (one asm block: the carry add stays a PREDICATED instruction; as C++ `if` it became a branch + reconvergence pair)
        asm volatile("{\n"
                     ".reg .pred p;\n"
                     ".reg .u32 o, t;\n"
                     "atom.shared.add.u32 o, [%0], %1;\n"
                     "add.u32 t, o, %1;\n"
                     "setp.lt.u32 p, t, o;\n"
                     "@p red.shared.add.u32 [%2], 1;\n"
                     "}\n" :: "r"(addr), "r"(q), "r"(addr + HIOFF) : "memory");
    };
    // deposits of one record into the accumulator (HM: the catalogue carries masses)
    auto deposit_record = [&](unsigned r0, unsigned r1, unsigned r2, MT mcur, auto hm_tag) {
            constexpr bool HM = decltype(hm_tag)::value;
            unsigned u[3] = {r0 << 4, r1 << 4, r2 << 4};
            int l[3] = {(int)(r0 >> 28), (int)(r1 >> 28), (int)(r2 >> 28)};
            double w[3][SUP];
#pragma unroll
            for (int d = 0; d < 3; d++) {
                if (SHIFTED) {                       // frac(g + A + 1/2): carry moves the stencil one cell up
                    unsigned v = u[d] + 0x80000000u;
                    l[d] += (v < u[d]) ? 1 : 0;
                    u[d] = v;
                }
                // u * 2^-32 via the 2^52 mantissa trick (no I2F)
                double fr = (__hiloint2double(0x43300000, (int)u[d]) - 4503599627370496.0) * 2.3283064365386963e-10;
                WinD<SUP>::eval(WinD<SUP>::DMIN != 0.0 ? WinD<SUP>::DMIN + fr : fr, w[d]);
            }
            const unsigned a0 = sbase + 4u * (unsigned)(l[0] * PS + l[1] * RP + l[2]);
            const double m = HM ? (double)mcur : 1.0;
            const double mS = m * S;
            double wz[SUP];
#pragma unroll
            for (int rz = 0; rz < SUP; rz++) wz[rz] = w[2][rz] * mS;
            if (!HM || m >= 0.0) {
                // all deposits are in [0, 2^31]: round-to-nearest integer = low word of fma(wxy, wz, 2^52)
#pragma unroll
                for (int rx = 0; rx < SUP; rx++)
#pragma unroll
                    for (int ry = 0; ry < SUP; ry++) {
                        const double wxy = w[0][rx] * w[1][ry];
                        const unsigned axy = a0 + 4u * (unsigned)(rx * PS + ry * RP);
#pragma unroll
                        for (int rz = 0; rz < SUP; rz++) {
                            const unsigned q = (unsigned)__double2loint(__fma_rn(wxy, wz[rz], 4503599627370496.0));
                            deposit(axy + 4u * (unsigned)rz, q);
                        }
                    }
            } else {
                const int base0 = l[0] * PS + l[1] * RP + l[2];       // negative weights: signed 64-bit deposits
#pragma unroll
                for (int rx = 0; rx < SUP; rx++)
#pragma unroll
                    for (int ry = 0; ry < SUP; ry++) {
                        const double wxy = w[0][rx] * w[1][ry];
#pragma unroll
                        for (int rz = 0; rz < SUP; rz++)
                            fixed_add(s_lo, s_hi, base0 + rx * PS + ry * RP + rz, __double2ll_rn(wxy * wz[rz]));
                    }
            }
    };
    // deposits of the records [b, e) of one bucket
    auto accumulate_recs = [&](unsigned b, unsigned e, auto hm_tag) {
        constexpr bool HM = decltype(hm_tag)::value;
        // thread p takes records p, p + NT, ... (coalesced)
        const unsigned cnt = e - b;
        unsigned idx = threadIdx.x;
        unsigned rn[3] = {0, 0, 0};
        MT mn = (MT)1;
        if (idx < cnt) {
            const unsigned *rp = recs + 3 * (size_t)(b + idx);
            rn[0] = rp[0]; rn[1] = rp[1]; rn[2] = rp[2];
            if (HM) mn = smass[b + idx];
        }
        for (; idx < cnt; idx += NT) {
            const unsigned r0 = rn[0], r1 = rn[1], r2 = rn[2];
            const MT mcur = mn;
            if (idx + NT < cnt) {                            // next round's record is requested before the deposits
                const unsigned *rp = recs + 3 * (size_t)(b + idx + NT);
                rn[0] = rp[0]; rn[1] = rp[1]; rn[2] = rp[2];
                if (HM) mn = smass[b + idx + NT];
            }
            deposit_record(r0, r1, r2, mcur, hm_tag);
        }
    };
    // deposits of the particles of the runs [b, e) of one bucket.  Warp w takes the runs b + 32 (w + 8 k) + lane (the
    // next 32 are requested before these are painted); over the particles of its 32 runs (exclusive scan of the lengths)
    // lane q takes particles q, q + 32, ...: the runs that start in a window of 32 particles form a bit mask (one
    // REDUX.OR), so the run of each lane is a popcount away, and consecutive lanes read consecutive particles of a run.
    auto accumulate_runs = [&](unsigned b, unsigned e, auto hm_tag) {
        if constexpr (RUNS) {
            constexpr bool HM = decltype(hm_tag)::value;
            unsigned eb = b + 32 * wid;
            uint2 rnext = make_uint2(0u, 0u);
            if (eb + lane < e) rnext = runs[recs[eb + lane]];
            for (; eb < e; eb += NT) {
                const bool valid = eb + lane < e;
                const unsigned len = valid ? (rnext.y & 127u) + 1u : 0u;
                const unsigned st = rnext.x;
                if (eb + NT + lane < e) rnext = runs[recs[eb + NT + lane]];
                unsigned inc = len;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const unsigned v = __shfl_up_sync(0xffffffffu, inc, o);
                    if ((int)lane >= o) inc += v;
                }
                const unsigned tot = __shfl_sync(0xffffffffu, inc, 31);
                const unsigned exc = inc - len;
                const unsigned base = st - exc;          // particle index = base + q for the q of this lane's run
                unsigned before = 0;                     // runs that start before the current window
                // particle index of this lane in the window [q0, q0 + 32); windows are taken in order; all lanes call
                auto particle = [&](unsigned q0) -> unsigned {
                    const unsigned m = __reduce_or_sync(0xffffffffu, (len && exc - q0 < 32u) ? 1u << (exc - q0) : 0u);
                    const int j = (int)before + __popc(m & ((2u << lane) - 1u)) - 1;
                    before += __popc(m);
                    return __shfl_sync(0xffffffffu, base, j & 31) + q0 + lane;
                };
                PT xn[3] = {(PT)0, (PT)0, (PT)0};
                MT mn = (MT)1;
                {
                    const unsigned i = particle(0);
                    if (lane < tot) {
                        xn[0] = pos[3 * (size_t)i]; xn[1] = pos[3 * (size_t)i + 1]; xn[2] = pos[3 * (size_t)i + 2];
                        if (HM) mn = smass[i];
                    }
                }
                for (unsigned q0 = 0; q0 < tot; q0 += 32) {
                    const PT x[3] = {xn[0], xn[1], xn[2]};
                    const MT mcur = mn;
                    if (q0 + 32 < tot) {                     // the next particle is requested before the deposits
                        const unsigned i = particle(q0 + 32);
                        if (q0 + 32 + lane < tot) {
                            xn[0] = pos[3 * (size_t)i]; xn[1] = pos[3 * (size_t)i + 1]; xn[2] = pos[3 * (size_t)i + 2];
                            if (HM) mn = smass[i];
                        }
                    }
                    if (q0 + lane < tot) {
                        unsigned r[3];
                        particle_record<SUP, PT>(x, tg, ft, r);
                        deposit_record(r[0], r[1], r[2], mcur, hm_tag);
                    }
                }
            }
        }
    };
    auto accumulate = [&](unsigned b, unsigned e) {
        if constexpr (RUNS) {
            if (smass) accumulate_runs(b, e, BoolTag<true>());
            else accumulate_runs(b, e, BoolTag<false>());
        } else {
            if (smass) accumulate_recs(b, e, BoolTag<true>());
            else accumulate_recs(b, e, BoolTag<false>());
        }
    };

    if (FLUSH == 1) {
        for (;;) {
            if (threadIdx.x == 0) s_tile = (int)atomicAdd(&hdr[HDR_QUEUE], 1u);
            __syncthreads();                                     // also: the accumulator is zero
            const int t = s_tile;
            if (t >= tg.ntiles) break;
            const unsigned b = offsets[t], e = offsets[t + 1];
            if (b == e) { __syncthreads(); continue; }
            accumulate(b, e);
            __syncthreads();
            const TileBox bx = tile_box<R, H>(t, tg);
            // ---- convert the region to mesh dtype (through registers: the values overlay the limb arrays), then one
            // TMA bulk reduce-add per z row
            constexpr int PER = (NC + NT - 1) / NT;
            FT v[PER];
#pragma unroll
            for (int k = 0; k < PER; k++) {
                int i = threadIdx.x + k * NT;
                v[k] = (FT)0;
                if (i < NC) v[k] = (FT)(limbs_to_double(s_lo[i], s_hi[i]) * invS);
            }
            __syncthreads();
#pragma unroll
            for (int k = 0; k < PER; k++) {
                int i = threadIdx.x + k * NT;
                if (i < NC) reinterpret_cast<FT *>(s_all)[i] = v[k];
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncthreads();
            const int nz1 = min(RP, tg.gm.n[2] - bx.o[2]);   // cells up to the end of the z row; the rest wraps to z = 0
            for (int row = threadIdx.x; row < R * R; row += NT) {
                int cx = row / R, cy = row - cx * R;
                int gx = bx.o[0] + cx + tg.gm.x_start;
                if (gx < 0) gx += tg.gm.n[0];
                if (gx >= tg.gm.n[0]) gx -= tg.gm.n[0];
                int ix = gx - tg.gm.x_start;
                if (ix < 0 || ix >= tg.gm.x_n) continue;     // not my plane (ghost semantics)
                int iy = bx.o[1] + cy; if (iy >= tg.gm.n[1]) iy -= tg.gm.n[1];
                FT *grow = mesh + ((int64_t)ix * tg.gm.n[1] + iy) * tg.gm.n[2];
                const FT *srow = reinterpret_cast<const FT *>(s_all) + (size_t)row * RP;
                tma_reduce_add(grow + bx.o[2], srow, (unsigned)(nz1 * sizeof(FT)));
                if (nz1 < RP) tma_reduce_add(grow, srow + nz1, (unsigned)((RP - nz1) * sizeof(FT)));
            }
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // shared memory may be reused
            __syncthreads();
            for (int i = threadIdx.x; i < BUFW / 4; i += NT) reinterpret_cast<uint4 *>(s_all)[i] = make_uint4(0, 0, 0, 0);
        }
        return;
    }

    // ================= ordered write-back =================
    // this thread's halo cells (tile independent): packed local coordinates, -1 = none
    int hcell[HK > 0 ? HK : 1];
    {
        constexpr int N1 = H * R * R, N2 = TILE * H * R;
        constexpr int HD = H > 0 ? H : 1;
#pragma unroll
        for (int k = 0; k < (HK > 0 ? HK : 1); k++) {
            const int i = (int)threadIdx.x + k * NT;
            int cx = 0, cy = 0, cz = 0;
            if (i < N1) { cx = TILE + i / (R * R); const int r = i % (R * R); cy = r / R; cz = r - cy * R; }
            else if (i < N1 + N2) { const int j = i - N1; cx = j / (HD * R); const int r = j - cx * (HD * R); cy = TILE + r / R; cz = r % R; }
            else { const int j = i - N1 - N2; cx = j / (TILE * HD); const int r = j - cx * (TILE * HD); cy = r / HD; cz = TILE + r % HD; }
            hcell[k] = (i < CAP) ? ((cx << 16) | (cy << 8) | cz) : -1;
        }
    }
    // every warp polls the flags of the (up to 26) earlier tiles overlapping tile `bx` itself: no CTA barrier
    auto poll_earlier = [&](const TileBox &bx) {
        if (lane < 27) {              // {this, following, wrapped-preceding} per axis
            int sel[3] = {(int)lane % 3, ((int)lane / 3) % 3, (int)lane / 9};
            int nb[3];
            bool valid = lane != 0;
#pragma unroll
            for (int d = 0; d < 3; d++) {
                if (sel[d] == 0) nb[d] = bx.tc[d];
                else if (sel[d] == 1) { nb[d] = bx.tc[d] + 1; valid = valid && bx.fhi[d] < R; }
                else { nb[d] = tg.nt[d] - 1; valid = valid && bx.flo[d] > 0 && bx.tc[d] != tg.nt[d] - 1; }
            }
            if (valid) {
                const unsigned *f = &flags[(nb[0] * tg.nt[1] + nb[1]) * tg.nt[2] + nb[2]];
                while (ld_relaxed(f) < epoch) __nanosleep(32);
            }
        }
        __syncwarp();
        fence_acq_rel_gpu();
    };
    // one look at the same flags, no waiting (warp-uniform result)
    auto earlier_ready = [&](const TileBox &bx) -> bool {
        bool ok = true;
        if (lane < 27) {
            int sel[3] = {(int)lane % 3, ((int)lane / 3) % 3, (int)lane / 9};
            int nb[3];
            bool valid = lane != 0;
#pragma unroll
            for (int d = 0; d < 3; d++) {
                if (sel[d] == 0) nb[d] = bx.tc[d];
                else if (sel[d] == 1) { nb[d] = bx.tc[d] + 1; valid = valid && bx.fhi[d] < R; }
                else { nb[d] = tg.nt[d] - 1; valid = valid && bx.flo[d] > 0 && bx.tc[d] != tg.nt[d] - 1; }
            }
            if (valid) ok = ld_relaxed(&flags[(nb[0] * tg.nt[1] + nb[1]) * tg.nt[2] + nb[2]]) >= epoch;
        }
        ok = __all_sync(0xffffffffu, ok);
        if (ok) fence_acq_rel_gpu();
        return ok;
    };
    // warp-aggregated append of (mesh offset, value) to the stash
    auto stash_push = [&](bool keep, unsigned off, FT val, unsigned *counter) {
        const unsigned mask = __ballot_sync(0xffffffffu, keep);
        if (mask) {
            unsigned basep = 0;
            const int leader = __ffs(mask) - 1;
            if ((int)lane == leader) basep = atomicAdd(counter, (unsigned)__popc(mask));
            basep = __shfl_sync(0xffffffffu, basep, leader);
            if (keep) {
                const unsigned pos = basep + __popc(mask & ((1u << lane) - 1u));
                s_soff[pos] = off;
                s_sval[pos] = val;
            }
        }
    };

    if (threadIdx.x == 0) s_tile = (int)atomicAdd(&hdr[HDR_QUEUE], 1u);
    __syncthreads();
    int t = tg.ntiles - 1 - s_tile;            // tiles are handed out in descending order
    bool pending = false;                      // the stash holds the add set of the previous tile (counter s_nst[pbuf])
    int pbuf = 0;
    TileBox pbox;
    for (;;) {
        // ---- (1) accumulate this tile, THEN add the parked set of the previous one: its neighbours had a whole
        // accumulation phase to publish, so the flag poll is almost never a wait
        if (t >= 0) accumulate(offsets[t], offsets[t + 1]);
        if (pending) {
            // The parked set goes onto blocks that EARLIER tiles store.  Normally they have published long ago; where one
            // has not (a dense neighbour still accumulating), the warp does not wait: it moves its share of the set to the
            // deferred list, which k_apply_deferred adds after this kernel.  (List full: wait as before.)
            const unsigned n = s_nst[pbuf];
            const bool ready = earlier_ready(pbox);
            bool defer = false;
            unsigned dbase = 0;
            if (!ready) {
                unsigned tot = 0;
                for (unsigned i0 = wid * 32; i0 < n; i0 += NT) tot += min(32u, n - i0);
                if (lane == 0 && tot) dbase = atomicAdd(&hdr[HDR_DEFER], tot);
                dbase = __shfl_sync(0xffffffffu, dbase, 0);
                defer = true;
                if (dbase + tot > d_cap || dbase + tot < dbase) {         // does not fit: neutral entries up to the cap, then wait
                    for (unsigned j = dbase + lane; j < d_cap && j - dbase < tot; j += 32) { d_off[j] = 0u; d_val[j] = (FT)0; }
                    defer = false;
                }
            }
            if (defer) {
                unsigned run = dbase;
                for (unsigned i0 = wid * 32; i0 < n; i0 += NT) {
                    const unsigned i = i0 + lane;
                    if (i < n) { d_off[run + lane] = s_soff[i]; d_val[run + lane] = s_sval[i]; }
                    run += min(32u, n - i0);
                }
            } else {
                if (!ready) poll_earlier(pbox);
                for (unsigned i = threadIdx.x; i < n; i += NT) atomicAdd(mesh + s_soff[i], s_sval[i]);
            }
        }
        if (t < 0) break;
        __syncthreads();                                                 // barrier 1 of 2
        const int cbuf = pbuf ^ 1;
        if (threadIdx.x == 0 && pending) s_nst[pbuf] = 0;                // consumed above by everyone
        pending = false;
        // ---- (3) write-back
        const TileBox bx = tile_box<R, H>(t, tg);
        const bool interior = small_mesh && bx.flo[0] == 0 && bx.flo[1] == 0 && bx.flo[2] == 0 &&
                              bx.fhi[0] == TILE && bx.fhi[1] == TILE && bx.fhi[2] == TILE;
        if (interior) {
            // base block: thread = (cy, z pair), 8 steps of two x planes; the accumulator is zeroed as it is read
            {
                const int row0 = (int)threadIdx.x >> 3, cz = ((int)threadIdx.x & 7) * 2;
                const int cy = row0 & 15, cx0 = row0 >> 4;
                int si = cx0 * PS + cy * RP + cz;
                int lx = bx.o[0] + cx0;                                   // slab-local x (full mesh: the global one)
                int64_t o64 = ((int64_t)lx * tg.gm.n[1] + (bx.o[1] + cy)) * tg.gm.n[2] + (bx.o[2] + cz);
                const int64_t ostep = 2 * (int64_t)tg.gm.n[1] * tg.gm.n[2];
#pragma unroll 4
                for (int j = 0; j < TILE / 2; j++) {
                    const uint2 lo2 = *reinterpret_cast<const uint2 *>(s_lo + si);
                    const uint2 hi2 = *reinterpret_cast<const uint2 *>(s_hi + si);
                    *reinterpret_cast<uint2 *>(s_lo + si) = make_uint2(0u, 0u);
                    *reinterpret_cast<uint2 *>(s_hi + si) = make_uint2(0u, 0u);
                    if (lx >= 0 && lx < tg.gm.x_n) {                      // ghost planes of a slab are dropped
                        const FT v0 = (FT)(limbs_to_double(lo2.x, hi2.x) * invS), v1 = (FT)(limbs_to_double(lo2.y, hi2.y) * invS);
                        if (sizeof(FT) == 8) *reinterpret_cast<double2 *>(mesh + o64) = make_double2((double)v0, (double)v1);
                        else *reinterpret_cast<float2 *>(mesh + o64) = make_float2((float)v0, (float)v1);
                    }
                    si += 2 * PS;
                    lx += 2;
                    o64 += ostep;
                }
            }
            // halo: parked (read, zeroed, appended to the stash)
#pragma unroll
            for (int k = 0; k < (HK > 0 ? HK : 1); k++) {
                bool keep = false;
                unsigned off = 0;
                FT val = (FT)0;
                if (HK > 0 && hcell[k] >= 0) {
                    const int cx = hcell[k] >> 16, cy = (hcell[k] >> 8) & 255, cz = hcell[k] & 255;
                    const int si = cx * PS + cy * RP + cz;
                    const unsigned lo = s_lo[si], hi = s_hi[si];
                    if ((lo | hi) != 0u) {
                        s_lo[si] = 0u;
                        s_hi[si] = 0u;
                        int lx = bx.o[0] + cx;
                        if (tg.full && lx >= tg.gm.n[0]) lx -= tg.gm.n[0];
                        if (lx >= 0 && lx < tg.gm.x_n) {
                            int iy = bx.o[1] + cy; if (iy >= tg.gm.n[1]) iy -= tg.gm.n[1];
                            int iz = bx.o[2] + cz; if (iz >= tg.gm.n[2]) iz -= tg.gm.n[2];
                            off = (unsigned)(((int64_t)lx * tg.gm.n[1] + iy) * tg.gm.n[2] + iz);
                            val = (FT)(limbs_to_double(lo, hi) * invS);
                            keep = true;
                        }
                    }
                }
                stash_push(keep, off, val, &s_nst[cbuf]);
            }
            pending = true;
        } else {
            // ---- mesh-boundary tiles: generic per-cell path
            const bool park = small_mesh && bx.flo[0] == 0 && bx.flo[1] == 0 && bx.flo[2] == 0;
            auto locate = [&](int cx, int cy, int cz, int64_t &o64) -> bool {
                int gx = bx.o[0] + cx + tg.gm.x_start;
                if (gx < 0) gx += tg.gm.n[0];
                if (gx >= tg.gm.n[0]) gx -= tg.gm.n[0];
                const int ix = gx - tg.gm.x_start;
                if (ix < 0 || ix >= tg.gm.x_n) return false;
                int iy = bx.o[1] + cy; if (iy >= tg.gm.n[1]) iy -= tg.gm.n[1];
                int iz = bx.o[2] + cz; if (iz >= tg.gm.n[2]) iz -= tg.gm.n[2];
                o64 = ((int64_t)ix * tg.gm.n[1] + iy) * tg.gm.n[2] + iz;
                return true;
            };
            // pass 0: store if this tile is first for the cell, else park it (or leave it to pass 1);
            // pass 1 (after the wait): add what was left
            auto sweep = [&](int pass) {
                for (int i0 = 0; i0 < R * R * R; i0 += NT) {
                    const int i = i0 + (int)threadIdx.x;
                    bool keep = false;
                    FT val = (FT)0;
                    unsigned off = 0;
                    if (i < R * R * R) {
                        const int cx = i / (R * R), r = i - cx * (R * R), cy = r / R, cz = r - cy * R;
                        const bool first = cx >= bx.flo[0] && cx < bx.fhi[0] && cy >= bx.flo[1] && cy < bx.fhi[1] &&
                                           cz >= bx.flo[2] && cz < bx.fhi[2];
                        int64_t o64;
                        if ((first == (pass == 0) || (pass == 0 && park)) && locate(cx, cy, cz, o64)) {
                            const int si = cx * PS + cy * RP + cz;
                            const unsigned lo = s_lo[si], hi = s_hi[si];
                            val = (FT)(limbs_to_double(lo, hi) * invS);
                            if (first) mesh[o64] = val;
                            else if ((lo | hi) != 0u) {
                                if (pass == 1) atomicAdd(mesh + o64, val);
                                else { keep = true; off = (unsigned)o64; }
                            }
                        }
                    }
                    if (pass == 0 && park) stash_push(keep, off, val, &s_nst[cbuf]);
                }
            };
            sweep(0);
            if (park) pending = true;
            else {
                __syncthreads();
                if (threadIdx.x == 0) st_release(&flags[t], epoch);
                poll_earlier(bx);
                sweep(1);
            }
            __syncthreads();
            for (int i = threadIdx.x; i < BUFW / 4; i += NT) reinterpret_cast<uint4 *>(s_all)[i] = make_uint4(0, 0, 0, 0);
        }
        // the next tile is taken only now: a tile that is handed out is also published one tile-time later, which is
        // what the tiles waiting on it count on
        if (threadIdx.x == 0) s_tile = (int)atomicAdd(&hdr[HDR_QUEUE], 1u);
        __syncthreads();                                                 // barrier 2 of 2
        if (threadIdx.x == 0) st_release(&flags[t], epoch);              // cumulative over the CTA's stores (bar.sync)
        if (pending) { pbox = bx; pbuf = cbuf; }
        t = tg.ntiles - 1 - s_tile;
    }
}

// adds the deferred halo sets (see k_tile_paint) once every tile has stored
template <typename FT>
__global__ void __launch_bounds__(256)
k_apply_deferred(const unsigned *__restrict__ hdr, const unsigned *__restrict__ d_off, const FT *__restrict__ d_val, unsigned d_cap,
                 FT *__restrict__ mesh) {
    unsigned n = hdr[HDR_DEFER];
    if (n > d_cap) n = d_cap;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const FT v = d_val[i];
        if (v != (FT)0) atomicAdd(mesh + d_off[i], v);
    }
}

static int make_tile_geom(const PaintGeom &gm, int sup, bool shifted, TileGeom &tg) {
    tg.gm = gm;
    tg.G = (gm.x_n == gm.n[0]) ? 0 : sup + 1;
    tg.full = (gm.x_n == gm.n[0] && gm.x_start == 0) ? 1 : 0;
    tg.R = TILE + sup - 1 + (shifted ? 1 : 0);
    tg.shifted = shifted ? 1 : 0;
    tg.nt[0] = (gm.x_n + tg.G + TILE - 1) / TILE;
    tg.nt[1] = (gm.n[1] + TILE - 1) / TILE;
    tg.nt[2] = (gm.n[2] + TILE - 1) / TILE;
    int64_t nt = (int64_t)tg.nt[0] * tg.nt[1] * tg.nt[2];
    NBK_CHECK_ARG(nt < (1ll << 30), "paint_tiled: too many tiles");
    tg.ntiles = (int)nt;
    return NBK_OK;
}

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

extern "C" int nbk_paint_tiled_supported(const int64_t *nmesh, int64_t x_n, int window) {
    int sup = window;
    if (sup < 1 || sup > 4) return 0;
    int R = TILE + sup;
    // the region must not wrap onto itself; tiles must not straddle the periodic seam (else a wrapped halo
    // would land in another tile's exclusively-owned cells); the slab must hold the ghost reach
    if (nmesh[1] < 2 * TILE || nmesh[2] < 2 * TILE || nmesh[0] < 2 * TILE || R > 2 * TILE) return 0;
    if (nmesh[1] % TILE || nmesh[2] % TILE) return 0;
    if (x_n == nmesh[0]) { if (nmesh[0] % TILE) return 0; }
    else if (x_n < sup + 1) return 0;
    return 1;
}

// the two bucketing configurations for a problem (only their sizes depend on it)
static int env_int(const char *name, int dflt) {
    const char *e = getenv(name);
    return (e && e[0]) ? atoi(e) : dflt;
}

static void plan_chunks(BucketPlan &p, int64_t n, int maxchunks) {
    int64_t nch = (n + 16383) / 16384;               // at least 16 Ki particles per chunk
    if (nch < 1) nch = 1;
    if (nch > maxchunks) nch = maxchunks;
    p.chunk = (((n + nch - 1) / nch) + 3) & ~(int64_t)3;   // multiple of 4: threads own aligned quads
    if (p.chunk < 4) p.chunk = 4;
    p.nchunks = (int)((n + p.chunk - 1) / p.chunk);
    if (p.nchunks < 1) p.nchunks = 1;
}

static void make_plans(int64_t n, const int *nt, int ntiles, BucketPlan &coh, BucketPlan &sca,
                       int &threads_coh, size_t &smem_coh, int &threads_sca, size_t &smem_sca) {
    auto align128 = [](size_t x) { return (x + 127) & ~(size_t)127; };
    // coherent input: a chunk spans a couple of planes of tiles (+- the displacement blur): 4 planes, at least 4096
    // tiles, at most NBK_WIN_COHERENT (64 KB)
    coh.mode = 1;
    int64_t w = 4 * (int64_t)nt[1] * nt[2];
    if (w < 4096) w = 4096;
    if (w > NBK_WIN_COHERENT) w = NBK_WIN_COHERENT;
    w = env_int("NBK_PAINT_W", (int)w);
    coh.W = ntiles < w ? ntiles : (int)w;
    plan_chunks(coh, n, NBK_CHUNKS_COHERENT);        // refined by the caller once the occupancy is known
    threads_coh = 512;                               // the size the coherent kernels are built for
    smem_coh = align128((size_t)coh.W * 4);
    coh.wstage = (env_int("NBK_PAINT_WSTAGE", 1) && n < 1400000000ll) ? 1 : 0;   // per-warp record transposition (2 KB per warp; 32-bit word offsets)
    coh.stage_off = (int)smem_coh;
    if (coh.wstage) smem_coh += (size_t)(threads_coh / 32) * 2048;
    sca.wstage = 0;                                                // scattered input: every record goes to another tile anyway
    sca.stage_off = 0;
    sca.mode = 0;
    sca.W = ntiles < NBK_BLK_SMEM / 4 ? ntiles : NBK_BLK_SMEM / 4;
    plan_chunks(sca, n, NBK_CHUNKS_SCATTERED);
    threads_sca = 1024;
    smem_sca = align128((size_t)sca.W * 4);
}

// capacity of the deferred-add list: a quarter of the tiles may park a full CIC halo (anything beyond waits instead)
static size_t nbk_defer_cap(int64_t ntiles) {
    size_t c = (size_t)ntiles * 208;
    if (c < (1u << 20)) c = 1u << 20;
    if (c > 0xfff00000u) c = 0xfff00000u;
    return c;
}

extern "C" int64_t nbk_paint_tiled_workspace(int64_t n, int pos_dtype, int mass_dtype, const int64_t *nmesh,
                                             int64_t x_n) {
    int64_t G = 8;
    int64_t nt = ((x_n + G + TILE - 1) / TILE) * ((nmesh[1] + TILE - 1) / TILE) * ((nmesh[2] + TILE - 1) / TILE);
    (void)pos_dtype;
    size_t bytes = 256;                                  // header: queue, absmax, mode
    bytes += 5 * align256(sizeof(unsigned) * (nt + 1));  // cnt_w, cnt_o, offsets, cur_o, flags
    bytes += align256(sizeof(unsigned) * ((size_t)(nt + 4095) / 4096 + 1));     // segment totals of the offset scan
    bytes += align256(sizeof(int) * NBK_CHUNKS_COHERENT);                // window start per chunk
    bytes += align256(sizeof(unsigned) * NBK_CHUNKS_COHERENT);           // runs per chunk (run plan)
    int64_t wc = nt < NBK_WIN_COHERENT ? nt : NBK_WIN_COHERENT, ws = nt < NBK_BLK_SMEM / 4 ? nt : NBK_BLK_SMEM / 4;
    int64_t blk = wc * NBK_CHUNKS_COHERENT > ws * NBK_CHUNKS_SCATTERED ? wc * NBK_CHUNKS_COHERENT : ws * NBK_CHUNKS_SCATTERED;
    bytes += align256(sizeof(unsigned) * (size_t)blk);                   // per-chunk bucket shares
    bytes += align256((size_t)n * 12);                                   // 12-byte records | run list (8 B) + run buckets (4 B)
    if (mass_dtype) bytes += align256((size_t)n * (mass_dtype == NBK_F4 ? 4 : 8));
    bytes += 2 * align256((size_t)nbk_defer_cap(nt) * 8);                // deferred halo adds: offsets (u32) and values (<= f8)
    return (int64_t)bytes;
}

template <int SUP, typename PT, typename MT, typename FT>
static int run_tiled(const void *pos, const void *mass, int64_t n, const PaintGeom &gm, double shift, void *mesh,
                     void *mesh2, void *work, bool clear, cudaStream_t s) {
    TileGeom tg;
    bool shifted = (mesh2 != nullptr) || shift != 0.0;
    int rc = make_tile_geom(gm, SUP, shifted, tg);
    if (rc) return rc;
    const FastTile ft = make_fast_tile(tg);
    char *w = (char *)work;
    unsigned *hdr = (unsigned *)w;
    w += 256;
    size_t tb = align256(sizeof(unsigned) * (tg.ntiles + 1));
    unsigned *cnt_w = (unsigned *)w; w += tb;
    unsigned *cnt_o = (unsigned *)w; w += tb;
    unsigned *offsets = (unsigned *)w; w += tb;
    unsigned *cur_o = (unsigned *)w; w += tb;
    unsigned *flags = (unsigned *)w; w += tb;
    unsigned *seg_tot = (unsigned *)w; w += align256(sizeof(unsigned) * ((size_t)(tg.ntiles + 4095) / 4096 + 1));   // scan: segment totals
    int *win_lo = (int *)w; w += align256(sizeof(int) * NBK_CHUNKS_COHERENT);
    unsigned *run_n = (unsigned *)w; w += align256(sizeof(unsigned) * NBK_CHUNKS_COHERENT);
    BucketPlan coh, sca;
    int th_c, th_s;
    size_t sm_c, sm_s;
    make_plans(n, tg.nt, tg.ntiles, coh, sca, th_c, sm_c, th_s, sm_s);
    unsigned *blk = (unsigned *)w;
    {
        size_t a = (size_t)coh.W * NBK_CHUNKS_COHERENT, b = (size_t)sca.W * NBK_CHUNKS_SCATTERED;
        w += align256(sizeof(unsigned) * (a > b ? a : b));
    }
    unsigned *recs = (unsigned *)w; w += align256((size_t)n * 12);
    uint2 *runs = reinterpret_cast<uint2 *>(recs);           // run plan: the run list and its buckets alias the records
    unsigned *rbucket = recs + 2 * (size_t)n;
    MT *smass = mass ? (MT *)w : nullptr;
    if (mass) w += align256((size_t)n * sizeof(MT));
    // NBK_PAINT_DEFER_CAP: smaller list (tests the overflow path)
    unsigned d_cap = (unsigned)nbk_defer_cap(tg.ntiles);
    {
        const int c = env_int("NBK_PAINT_DEFER_CAP", 0);
        if (c > 0 && (unsigned)c < d_cap) d_cap = (unsigned)c;
    }
    unsigned *d_off = (unsigned *)w; w += align256((size_t)nbk_defer_cap(tg.ntiles) * 8);
    FT *d_val = (FT *)w; w += align256((size_t)nbk_defer_cap(tg.ntiles) * 8);
    const int mass_f4 = sizeof(MT) == 4;
    // The run plan packs the tile id into RUN_TILE_BITS bits.  Its tile pass rebuilds every record, once per mesh: the
    // probe picks it for one NNB / CIC mesh, where that costs less than the record stream saves (DESIGN.md 4.1); TSC /
    // PCS and the interlaced pair keep the record plans unless NBK_PAINT_BUCKET=runs forces it.
    const int runs_ok = tg.ntiles <= (1 << RUN_TILE_BITS);
    const int runs_auto = runs_ok && SUP <= 2 && mesh2 == nullptr;
    int force_mode;
    {
        const char *e = getenv("NBK_PAINT_BUCKET");      // "coherent" / "scattered" / "runs" force the configuration the probe picks
        force_mode = (e && e[0] == 'c') ? 1 : (e && e[0] == 's') ? 0 : (e && e[0] == 'r') ? 2 : -1;
    }
    NBK_CHECK_ARG(force_mode != 2 || runs_ok, "paint_tiled: NBK_PAINT_BUCKET=runs needs at most 2^%d tiles", RUN_TILE_BITS);
    const bool runs_on = force_mode == 2 || (force_mode < 0 && runs_auto);     // the run kernels are launched
    NBK_CUDA(cudaMemsetAsync(work, 0, 256 + 2 * tb, s));   // header, cnt_w, cnt_o
    if (force_mode >= 0) {
        unsigned m = (unsigned)force_mode;
        NBK_CUDA(cudaMemcpyAsync(&hdr[HDR_MODE], &m, sizeof(unsigned), cudaMemcpyHostToDevice, s));
    } else {
        k_bucket_probe<SUP, PT><<<1, 256, 0, s>>>((const PT *)pos, n, tg, runs_auto, hdr);
        NBK_LAUNCHED();
    }
    // Coherent plan: every resident CTA gets the same number of chunks in BOTH passes (their occupancies differ:
    // the scatter pass needs more registers), else the last partial wave runs at a fraction of the machine.
    int occ_c = 1, occ_s = 1;
    const size_t sm_cnt = coh.wstage ? (size_t)coh.stage_off : sm_c;      // the count pass does not need the record staging
    NBK_CUDA(cudaFuncSetAttribute(k_bucket_count<SUP, PT, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_c));
    NBK_CUDA(cudaFuncSetAttribute(k_bucket_scatter<SUP, PT, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_c));
    NBK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_c, k_bucket_count<SUP, PT, 512>, th_c, sm_cnt));
    NBK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_s, k_bucket_scatter<SUP, PT, 512>, th_c, sm_c));
    if (occ_c < 1) occ_c = 1;
    if (occ_s < 1) occ_s = 1;
    if (occ_c > 4) occ_c = 4;
    if (occ_s > 4) occ_s = 4;
    {
        int l = occ_c * occ_s, a = occ_c, b = occ_s;
        while (b) { int r = a % b; a = b; b = r; }
        l /= a;                                              // lcm <= 12
        plan_chunks(coh, n, l * NBK_SM_COUNT);
    }
    const int grid_c = coh.nchunks < occ_c * NBK_SM_COUNT ? coh.nchunks : occ_c * NBK_SM_COUNT;
    const int grid_cs = coh.nchunks < occ_s * NBK_SM_COUNT ? coh.nchunks : occ_s * NBK_SM_COUNT;
    const int grid_s = sca.nchunks < NBK_SM_COUNT ? sca.nchunks : NBK_SM_COUNT;
#define LAUNCH_BUCKET(KERN, GRIDC, SMC, ...)                                                                                      \
    do {                                                                                                              \
        NBK_CUDA(cudaFuncSetAttribute(KERN<SUP, PT, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(SMC)));  \
        KERN<SUP, PT, 512><<<GRIDC, th_c, SMC, s>>>(__VA_ARGS__, coh);                                                \
        NBK_LAUNCHED();                                                                                               \
        NBK_CUDA(cudaFuncSetAttribute(KERN<SUP, PT, 1024>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_s));  \
        KERN<SUP, PT, 1024><<<grid_s, th_s, sm_s, s>>>(__VA_ARGS__, sca);                                             \
        NBK_LAUNCHED();                                                                                               \
    } while (0)
    // (the plan is the LAST kernel argument of both passes so that one macro serves them)
    LAUNCH_BUCKET(k_bucket_count, grid_c, sm_cnt, (const PT *)pos, mass, mass_f4, n, tg, ft, hdr, cnt_w, cnt_o, blk, win_lo);
    // run plan: the coherent plan's chunks and window
    BucketPlan rp = coh;
    rp.mode = 2;
    rp.wstage = 0;
    const size_t sm_run = (size_t)coh.W * 4;
    int grid_rc = 1, grid_rp = 1;
    if (runs_on) {
        NBK_CUDA(cudaFuncSetAttribute(k_run_count<SUP, PT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_run));
        NBK_CUDA(cudaFuncSetAttribute(k_run_place, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_run));
        int occ_rc = 1, occ_rp = 1;
        NBK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_rc, k_run_count<SUP, PT>, 512, sm_run));
        NBK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_rp, k_run_place, 512, sm_run));
        grid_rc = rp.nchunks < max(occ_rc, 1) * NBK_SM_COUNT ? rp.nchunks : max(occ_rc, 1) * NBK_SM_COUNT;
        grid_rp = rp.nchunks < max(occ_rp, 1) * NBK_SM_COUNT ? rp.nchunks : max(occ_rp, 1) * NBK_SM_COUNT;
        k_run_count<SUP, PT><<<grid_rc, 512, sm_run, s>>>((const PT *)pos, mass, mass_f4, n, tg, ft, hdr, cnt_w, cnt_o, blk,
                                                         win_lo, runs, run_n, rp);
        NBK_LAUNCHED();
    }
    {
        const int nseg = (tg.ntiles + 4095) / 4096;
        k_tile_scan_totals<<<nseg, 1024, 0, s>>>(cnt_w, cnt_o, seg_tot, tg.ntiles);
        NBK_LAUNCHED();
        k_tile_scan<<<nseg, 1024, 0, s>>>(cnt_w, cnt_o, seg_tot, offsets, cur_o, flags, hdr, tg.ntiles);
        NBK_LAUNCHED();
    }
    LAUNCH_BUCKET(k_bucket_scatter, grid_cs, sm_c, (const PT *)pos, mass, mass_f4, n, tg, ft, hdr, offsets, cnt_w, cur_o, blk, win_lo, recs,
                  (void *)smass);
#undef LAUNCH_BUCKET
    if (runs_on) {
        k_run_place<<<grid_rp, 512, sm_run, s>>>(runs, run_n, tg.ntiles, hdr, offsets, cnt_w, cur_o, blk, win_lo, rbucket, rp);
        NBK_LAUNCHED();
    }
    // the region edge depends on the mesh being painted (one more cell for the half-cell shifted one); tile ids do not.
    // Both sources are launched (the one the probe did not pick exits at once), then one pass adds the deferred sets.
#define LAUNCH_TP1(SH, FL, MESHP, EPOCH, SRC, RECS, MASS)                                                              \
    do {                                                                                                              \
        const int Rr = TILE + SUP - 1 + ((SH) ? 1 : 0), RPr = (FL) == 0 ? ((Rr + 1) & ~1) : ((Rr + 3) & ~3);         \
        size_t smem = (size_t)((2 * Rr * tile_plane_pitch(SUP, FL, Rr, RPr) + 3) & ~3) * sizeof(unsigned);            \
        if ((FL) == 0) smem += (size_t)(Rr * Rr * Rr - TILE * TILE * TILE) * (sizeof(FT) + sizeof(unsigned));        \
        NBK_CUDA(cudaFuncSetAttribute(k_tile_paint<SUP, MT, FT, SH, FL, SRC>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                      (int)smem));                                                                    \
        int per_sm = 1;                                                                                               \
        NBK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_tile_paint<SUP, MT, FT, SH, FL, SRC>, 256, smem)); \
        if (per_sm < 1) per_sm = 1;                                                                                   \
        int grid = NBK_SM_COUNT * per_sm;                                                                             \
        if (grid > tg.ntiles) grid = tg.ntiles;                                                                       \
        k_tile_paint<SUP, MT, FT, SH, FL, SRC><<<grid, 256, smem, s>>>(RECS, MASS, tg, offsets, hdr, flags, EPOCH,    \
                                                                       (FT *)(MESHP), d_off, d_val, d_cap, runs,      \
                                                                       (const SRC *)pos, ft);                        \
        NBK_LAUNCHED();                                                                                               \
    } while (0)
#define LAUNCH_TP(SH, FL, MESHP, EPOCH)                                                                                \
    do {                                                                                                              \
        LAUNCH_TP1(SH, FL, MESHP, EPOCH, void, recs, smass);                                                         \
        if (runs_on) LAUNCH_TP1(SH, FL, MESHP, EPOCH, PT, rbucket, (const MT *)mass);                                \
        if ((FL) == 0) {                                                                                              \
            k_apply_deferred<FT><<<NBK_SM_COUNT * 4, 256, 0, s>>>(hdr, d_off, d_val, d_cap, (FT *)(MESHP));           \
            NBK_LAUNCHED();                                                                                           \
        }                                                                                                             \
    } while (0)
    if (shift != 0.0) { if (clear) LAUNCH_TP(true, 0, mesh, 1u); else LAUNCH_TP(true, 1, mesh, 1u); }
    else { if (clear) LAUNCH_TP(false, 0, mesh, 1u); else LAUNCH_TP(false, 1, mesh, 1u); }
    if (mesh2) {
        NBK_CUDA(cudaMemsetAsync(&hdr[HDR_QUEUE], 0, sizeof(unsigned), s));
        NBK_CUDA(cudaMemsetAsync(&hdr[HDR_DEFER], 0, sizeof(unsigned), s));
        if (clear) LAUNCH_TP(true, 0, mesh2, 2u); else LAUNCH_TP(true, 1, mesh2, 2u);
    }
#undef LAUNCH_TP1
#undef LAUNCH_TP
    return NBK_OK;
}

template <int SUP, typename PT, typename MT>
static int run_tiled1(const void *pos, const void *mass, int64_t n, const PaintGeom &gm, double shift, void *mesh,
                      void *mesh2, int mesh_dtype, void *work, bool clear, cudaStream_t s) {
    if (mesh_dtype == NBK_F4) return run_tiled<SUP, PT, MT, float>(pos, mass, n, gm, shift, mesh, mesh2, work, clear, s);
    return run_tiled<SUP, PT, MT, double>(pos, mass, n, gm, shift, mesh, mesh2, work, clear, s);
}

template <int SUP>
static int run_tiled0(const void *pos, int pos_dtype, const void *mass, int mass_dtype, int64_t n, const PaintGeom &gm,
                      double shift, void *mesh, void *mesh2, int mesh_dtype, void *work, bool clear, cudaStream_t s) {
    bool pf4 = pos_dtype == NBK_F4, mf4 = (mass_dtype == NBK_F4);
    if (pf4 && mf4) return run_tiled1<SUP, float, float>(pos, mass, n, gm, shift, mesh, mesh2, mesh_dtype, work, clear, s);
    if (pf4) return run_tiled1<SUP, float, double>(pos, mass, n, gm, shift, mesh, mesh2, mesh_dtype, work, clear, s);
    if (mf4) return run_tiled1<SUP, double, float>(pos, mass, n, gm, shift, mesh, mesh2, mesh_dtype, work, clear, s);
    return run_tiled1<SUP, double, double>(pos, mass, n, gm, shift, mesh, mesh2, mesh_dtype, work, clear, s);
}

extern "C" int nbk_paint_tiled(const void *pos, int pos_dtype, int64_t n, const void *mass, int mass_dtype, int window,
                               double shift, const double *box, const int64_t *nmesh, int64_t x_start, int64_t x_n,
                               void *mesh, void *mesh2, int mesh_dtype, void *work, int64_t work_bytes, int clear,
                               void *stream) {
    NBK_CHECK_ARG(pos_dtype == NBK_F4 || pos_dtype == NBK_F8, "paint_tiled: bad pos dtype %d", pos_dtype);
    NBK_CHECK_ARG(mesh_dtype == NBK_F4 || mesh_dtype == NBK_F8, "paint_tiled: bad mesh dtype %d", mesh_dtype);
    NBK_CHECK_ARG(mass == nullptr || mass_dtype == NBK_F4 || mass_dtype == NBK_F8, "paint_tiled: bad mass dtype %d", mass_dtype);
    NBK_CHECK_ARG(n >= 0 && n < (1ll << 32) - 1024, "paint_tiled: particle count %lld out of range", (long long)n);
    NBK_CHECK_ARG(mesh != nullptr && work != nullptr, "paint_tiled: null mesh / workspace");
    NBK_CHECK_ARG(mesh2 == nullptr || shift == 0.0, "paint_tiled: the interlaced pair is painted with shifts (0, 0.5)");
    NBK_CHECK_ARG(shift == 0.0 || shift == 0.5, "paint_tiled: shift must be 0 or 0.5 cells");
    NBK_CHECK_ARG(nbk_paint_tiled_supported(nmesh, x_n, window), "paint_tiled: mesh too small for the tiled path (use nbk_paint)");
    PaintGeom gm;
    int rc = make_geom(box, nmesh, x_start, x_n, gm);
    if (rc) return rc;
    if (x_n == 0) return NBK_OK;
    if (n == 0) {
        if (clear) {
            size_t mb = (size_t)x_n * nmesh[1] * nmesh[2] * (mesh_dtype == NBK_F4 ? 4 : 8);
            NBK_CUDA(cudaMemsetAsync(mesh, 0, mb, (cudaStream_t)stream));
            if (mesh2) NBK_CUDA(cudaMemsetAsync(mesh2, 0, mb, (cudaStream_t)stream));
        }
        return NBK_OK;
    }
    int md = mass ? mass_dtype : 0;
    NBK_CHECK_ARG(work_bytes >= nbk_paint_tiled_workspace(n, pos_dtype, md, nmesh, x_n), "paint_tiled: workspace too small");
    if (mass == nullptr) mass_dtype = NBK_F8;
    cudaStream_t s = (cudaStream_t)stream;
    switch (window) {
        case NBK_WINDOW_NNB: return run_tiled0<1>(pos, pos_dtype, mass, mass_dtype, n, gm, shift, mesh, mesh2, mesh_dtype, work, clear != 0, s);
        case NBK_WINDOW_CIC: return run_tiled0<2>(pos, pos_dtype, mass, mass_dtype, n, gm, shift, mesh, mesh2, mesh_dtype, work, clear != 0, s);
        case NBK_WINDOW_TSC: return run_tiled0<3>(pos, pos_dtype, mass, mass_dtype, n, gm, shift, mesh, mesh2, mesh_dtype, work, clear != 0, s);
        case NBK_WINDOW_PCS: return run_tiled0<4>(pos, pos_dtype, mass, mass_dtype, n, gm, shift, mesh, mesh2, mesh_dtype, work, clear != 0, s);
    }
    nbk_set_error("paint_tiled: unknown window %d", window);
    return NBK_ERR_ARG;
}

extern "C" int nbk_paint(const void *pos, int pos_dtype, int64_t n, const void *mass, int mass_dtype, int window,
                         double shift, const double *box, const int64_t *nmesh, int64_t x_start, int64_t x_n,
                         void *mesh, int mesh_dtype, void *stream) {
    return paint_impl(pos, pos_dtype, n, mass, mass_dtype, window, shift, box, nmesh, x_start, x_n, mesh, nullptr,
                      mesh_dtype, stream);
}

extern "C" int nbk_paint_interlaced(const void *pos, int pos_dtype, int64_t n, const void *mass, int mass_dtype,
                                    int window, const double *box, const int64_t *nmesh, int64_t x_start,
                                    int64_t x_n, void *mesh1, void *mesh2, int mesh_dtype, void *stream) {
    NBK_CHECK_ARG(mesh2 != nullptr, "paint_interlaced: null mesh2");
    return paint_impl(pos, pos_dtype, n, mass, mass_dtype, window, 0.0, box, nmesh, x_start, x_n, mesh1, mesh2,
                      mesh_dtype, stream);
}

extern "C" int nbk_cell_index(const void *pos, int pos_dtype, int64_t n, int window, double shift, const double *box,
                              const int64_t *nmesh, int32_t *cell_out, void *stream) {
    NBK_CHECK_ARG(pos_dtype == NBK_F4 || pos_dtype == NBK_F8, "cell_index: bad pos dtype %d", pos_dtype);
    PaintGeom gm;
    int rc = make_geom(box, nmesh, 0, nmesh[0], gm);
    if (rc) return rc;
    if (n == 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    int g = nbk_grid_for(n, 256, 8);
#define CI(SUP)                                                                                              \
    if (pos_dtype == NBK_F4) k_cell_index<SUP, float><<<g, 256, 0, s>>>((const float *)pos, n, gm, shift, cell_out); \
    else k_cell_index<SUP, double><<<g, 256, 0, s>>>((const double *)pos, n, gm, shift, cell_out);
    switch (window) {
        case NBK_WINDOW_NNB: CI(1); break;
        case NBK_WINDOW_CIC: CI(2); break;
        case NBK_WINDOW_TSC: CI(3); break;
        case NBK_WINDOW_PCS: CI(4); break;
        default: nbk_set_error("cell_index: unknown window %d", window); return NBK_ERR_ARG;
    }
#undef CI
    NBK_LAUNCHED();
    return NBK_OK;
}

// =============================================================================================
// readout (gather): value_p = sum over the stencil of W * mesh[cell] -- pmesh `RealField.readout`, the transpose of the
// scatter above (algorithms/fftrecon.py:239-244 reads the displacement field at the particle positions).  Same grid
// coordinate, window and slab semantics as `scatter`: planes outside [x_start, x_start + x_n) contribute nothing,
// so with x slabs every rank produces the partial sum of its own planes.  One particle per thread, support^3 cached
// loads, f8 accumulation in the order (x, y, z) of the stencil.
// =============================================================================================
template <int SUP, typename PT, typename FT, typename OT>
__global__ void __launch_bounds__(256)
k_readout(const PT *__restrict__ pos, int64_t n, PaintGeom gm, double shift, const FT *__restrict__ mesh,
          OT *__restrict__ out, int accumulate) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        double g[3];
        double acc = 0.0;
        if (load_grid(pos, i, gm, shift, g)) {
            long long i0[3];
            double w[3][SUP];
#pragma unroll
            for (int d = 0; d < 3; d++) Window<SUP>::eval(g[d], i0[d], w[d]);
            int iz[SUP], iy[SUP];
#pragma unroll
            for (int r = 0; r < SUP; r++) {
                iz[r] = wrap(i0[2] + r, gm.n[2]);
                iy[r] = wrap(i0[1] + r, gm.n[1]);
            }
#pragma unroll
            for (int rx = 0; rx < SUP; rx++) {
                int ix = wrap(i0[0] + rx, gm.n[0]) - gm.x_start;
                if (ix < 0 || ix >= gm.x_n) continue;
#pragma unroll
                for (int ry = 0; ry < SUP; ry++) {
                    double wxy = w[0][rx] * w[1][ry];
                    int64_t row = ((int64_t)ix * gm.n[1] + iy[ry]) * gm.n[2];
#pragma unroll
                    for (int rz = 0; rz < SUP; rz++) acc += (wxy * w[2][rz]) * (double)mesh[row + iz[rz]];
                }
            }
        }
        out[i] = accumulate ? (OT)((double)out[i] + acc) : (OT)acc;
    }
}

template <int SUP>
static int launch_readout(const void *pos, int pos_dtype, int64_t n, const PaintGeom &gm, double shift, const void *mesh,
                          int mesh_dtype, void *out, int out_dtype, int accumulate, cudaStream_t s) {
    int g = nbk_grid_for(n, 256, 8);
#define RO(PT, FT, OT) k_readout<SUP, PT, FT, OT><<<g, 256, 0, s>>>((const PT *)pos, n, gm, shift, (const FT *)mesh, (OT *)out, accumulate)
    const bool pf = pos_dtype == NBK_F4, ff = mesh_dtype == NBK_F4, of = out_dtype == NBK_F4;
    if (pf) { if (ff) { if (of) RO(float, float, float); else RO(float, float, double); }
              else { if (of) RO(float, double, float); else RO(float, double, double); } }
    else { if (ff) { if (of) RO(double, float, float); else RO(double, float, double); }
           else { if (of) RO(double, double, float); else RO(double, double, double); } }
#undef RO
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_readout(const void *mesh, int mesh_dtype, const void *pos, int pos_dtype, int64_t n, int window,
                           double shift, const double *box, const int64_t *nmesh, int64_t x_start, int64_t x_n,
                           void *out, int out_dtype, int accumulate, void *stream) {
    NBK_CHECK_ARG(pos_dtype == NBK_F4 || pos_dtype == NBK_F8, "readout: bad pos dtype %d", pos_dtype);
    NBK_CHECK_ARG(mesh_dtype == NBK_F4 || mesh_dtype == NBK_F8, "readout: bad mesh dtype %d", mesh_dtype);
    NBK_CHECK_ARG(out_dtype == NBK_F4 || out_dtype == NBK_F8, "readout: bad out dtype %d", out_dtype);
    NBK_CHECK_ARG(n >= 0 && mesh != nullptr && (n == 0 || out != nullptr), "readout: null mesh / out or negative count");
    PaintGeom gm;
    int rc = make_geom(box, nmesh, x_start, x_n, gm);
    if (rc) return rc;
    if (n == 0) return NBK_OK;
    cudaStream_t s = (cudaStream_t)stream;
    switch (window) {
        case NBK_WINDOW_NNB: return launch_readout<1>(pos, pos_dtype, n, gm, shift, mesh, mesh_dtype, out, out_dtype, accumulate, s);
        case NBK_WINDOW_CIC: return launch_readout<2>(pos, pos_dtype, n, gm, shift, mesh, mesh_dtype, out, out_dtype, accumulate, s);
        case NBK_WINDOW_TSC: return launch_readout<3>(pos, pos_dtype, n, gm, shift, mesh, mesh_dtype, out, out_dtype, accumulate, s);
        case NBK_WINDOW_PCS: return launch_readout<4>(pos, pos_dtype, n, gm, shift, mesh, mesh_dtype, out, out_dtype, accumulate, s);
    }
    nbk_set_error("readout: unknown window %d", window);
    return NBK_ERR_ARG;
}
