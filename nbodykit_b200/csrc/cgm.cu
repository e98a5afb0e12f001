// Cylindrical groups of centrals and satellites (nbodykit/algorithms/cgm.py: CylindricalGroups; DESIGN.md 4.9) on the
// cell grid of csrc/fof.cu and the neighbour walk of pc_cells.cuh.
//   nbk_cgm_count   : per owned row i, the number of rows j linked to it with prio_j > prio_i
//   nbk_cgm_write   : the same walk again, writing those j (sorted row indices) into i's CSR list
//   nbk_cgm_resolve : one round of the greedy: an undecided row becomes a satellite when one of its higher-priority
//                     neighbours is a central, a central when all of them are satellites (or it has none)
//   nbk_cgm_assign  : every satellite takes the highest-priority central among its higher-priority neighbours
// Link of rows a != b, a the higher-priority row, all in double from the stored (wrapped) positions:
//   dr = x_a - x_b per axis (periodic: dr > L/2 -> dr - L, dr <= -L/2 -> dr + L), dr2 = (dx^2 + dy^2) + dz^2,
//   flat sky: t = (dx lx + dy ly) + dz lz, rlos2 = t^2;
//   otherwise c = 0.5 (x_a + x_b), t = (dx cx + dy cy) + dz cz, rlos2 = t^2 / ((cx^2 + cy^2) + cz^2), unlinked when that
//   denominator is 0;  rsky2 = |dr2 - rlos2|;  linked iff rsky2 <= rperp^2 and rlos2 <= rpar^2.
// The file is compiled with --fmad=false: no contraction may move a pair across the cylinder's edge.
#include "pc_cells.cuh"

#include <math.h>

#define CGM_B 128
#define CGM_RB 256
#define CGM_MAX_CELLS_PER_AXIS (1ll << 21)

#define CGM_UNDECIDED 0
#define CGM_CENTRAL 1
#define CGM_SATELLITE 2

struct CgmLink {
    double los[3];
    double rperp2, rpar2;
};

template <bool FLAT>
static __device__ __forceinline__ bool cgm_linked(double ax, double ay, double az, double bx, double by, double bz,
                                                  const PcGeom &g, const CgmLink &k) {
    double dx = ax - bx, dy = ay - by, dz = az - bz;
    if (g.periodic) {
        const double hx = 0.5 * g.box[0], hy = 0.5 * g.box[1], hz = 0.5 * g.box[2];
        if (dx > hx) dx -= g.box[0]; else if (dx <= -hx) dx += g.box[0];
        if (dy > hy) dy -= g.box[1]; else if (dy <= -hy) dy += g.box[1];
        if (dz > hz) dz -= g.box[2]; else if (dz <= -hz) dz += g.box[2];
    }
    const double dr2 = (dx * dx + dy * dy) + dz * dz;
    double rlos2;
    if (FLAT) {
        const double t = (dx * k.los[0] + dy * k.los[1]) + dz * k.los[2];
        rlos2 = t * t;
    } else {
        const double cx = 0.5 * (ax + bx), cy = 0.5 * (ay + by), cz = 0.5 * (az + bz);
        const double den = (cx * cx + cy * cy) + cz * cz;
        if (!(den > 0.0)) return false;
        const double t = (dx * cx + dy * cy) + dz * cz;
        rlos2 = (t * t) / den;
    }
    const double rsky2 = fabs(dr2 - rlos2);
    return rsky2 <= k.rperp2 && rlos2 <= k.rpar2;
}

// One CTA per chunk of at most CGM_B primaries of one cell; the rows of every neighbour column are staged through shared
// memory in tiles of CGM_B.  WRITE = false: cnt[i] = number of higher-priority neighbours of sorted row i (owned rows
// only, 0 for copies).  WRITE = true: those neighbours, in walk order, at nbr[off[i] ..].
template <bool WRITE, bool FLAT>
__global__ void __launch_bounds__(CGM_B, 4) k_cgm_walk(const double *__restrict__ spos, const long long *__restrict__ sprio,
                                                      const unsigned *__restrict__ perm, long long n_own,
                                                      const long long *__restrict__ chunk_first, const long long *__restrict__ chunk_key,
                                                      const unsigned *__restrict__ cell_start, const long long *__restrict__ cell_key,
                                                      int64_t ncells, PcGeom g, CgmLink lk, long long *__restrict__ cnt,
                                                      const long long *__restrict__ off, int *__restrict__ nbr,
                                                      unsigned long long *__restrict__ g_cand) {
    __shared__ double tile[3 * CGM_B];
    __shared__ long long tprio[CGM_B];
    const int64_t c = blockIdx.x;
    const long long p0 = chunk_first[c], np = chunk_first[c + 1] - p0;
    const long long key = chunk_key[c];
    const long long nyz = g.nc[1] * g.nc[2];
    const long long ix = key / nyz, iy = (key / g.nc[2]) % g.nc[1], iz = key % g.nc[2];
    const long long i = p0 + threadIdx.x;
    const bool have = threadIdx.x < np && (long long)perm[i] < n_own;
    double px = 0.0, py = 0.0, pz = 0.0;
    long long pp = 0, found = 0, w = 0;
    if (have) {
        px = spos[3 * i]; py = spos[3 * i + 1]; pz = spos[3 * i + 2];
        pp = sprio[i];
        if (WRITE) w = off[i];
    }
    unsigned long long cand = 0;

    const PcAxis ax = pc_axis(ix, g.reach[0], 0, g), ay = pc_axis(iy, g.reach[1], 1, g);
    for (long long xx = ax.lo; xx <= ax.hi; xx++) {
        const long long x = g.periodic ? pc_wrap(xx, g.nc[0]) : xx;
        const double gx = axis_gap(pc_delta(xx, ix, ax.all, g.nc[0]), 0, g);
        for (long long yy = ay.lo; yy <= ay.hi; yy++) {
            const long long y = g.periodic ? pc_wrap(yy, g.nc[1]) : yy;
            const double gy = axis_gap(pc_delta(yy, iy, ay.all, g.nc[1]), 1, g);
            const double gxy2 = gx * gx + gy * gy;
            if (gxy2 >= g.thr_sph) continue;
            // the z cells this column can still reach: gap_z < rem
            const double rem = sqrt(g.thr_sph - gxy2);
            const double rzd = floor((rem + g.tol[2]) / g.cs[2]) + 1.0;
            const long long rz = rzd < (double)g.reach[2] ? (long long)rzd : g.reach[2];
            const PcAxis az = pc_axis(iz, rz, 2, g);
            long long z0[2], z1[2];
            int nr = 0;
            if (az.all || !g.periodic) { z0[nr] = az.lo; z1[nr++] = az.hi; }
            else if (az.lo < 0) { z0[nr] = az.lo + g.nc[2]; z1[nr++] = g.nc[2] - 1; z0[nr] = 0; z1[nr++] = az.hi; }
            else if (az.hi >= g.nc[2]) { z0[nr] = az.lo; z1[nr++] = g.nc[2] - 1; z0[nr] = 0; z1[nr++] = az.hi - g.nc[2]; }
            else { z0[nr] = az.lo; z1[nr++] = az.hi; }
            const long long row = (x * g.nc[1] + y) * g.nc[2];
            for (int q = 0; q < nr; q++) {
                const int64_t d0 = pc_lower_bound(cell_key, ncells, row + z0[q]);
                const int64_t d1 = pc_lower_bound(cell_key, ncells, row + z1[q] + 1);
                if (d0 >= d1) continue;
                const long long r0 = cell_start[d0], r1 = cell_start[d1];
                for (long long base = r0; base < r1; base += CGM_B) {
                    const int m = (int)(r1 - base < CGM_B ? r1 - base : CGM_B);
                    __syncthreads();
                    if (threadIdx.x < m) {
                        const long long r = base + threadIdx.x;
                        tile[threadIdx.x] = spos[3 * r];
                        tile[CGM_B + threadIdx.x] = spos[3 * r + 1];
                        tile[2 * CGM_B + threadIdx.x] = spos[3 * r + 2];
                        tprio[threadIdx.x] = sprio[r];
                    }
                    __syncthreads();
                    cand += (unsigned long long)m;
                    if (!have) continue;
                    for (int j = 0; j < m; j++) {
                        if (tprio[j] <= pp) continue;
                        if (!cgm_linked<FLAT>(tile[j], tile[CGM_B + j], tile[2 * CGM_B + j], px, py, pz, g, lk)) continue;
                        if (WRITE) nbr[w + found] = (int)(base + j);
                        found++;
                    }
                }
            }
        }
    }
    if (have && !WRITE) cnt[i] = found;
    if (threadIdx.x == 0 && !WRITE) atomicAdd(g_cand, cand * (unsigned long long)np);
}

// One round.  Rows in descending priority, 32 per warp; a warp repeats while any of its lanes decides.  A decision reads
// final states only, and states only move from undecided to final, so the in-place updates need no ordering.
__global__ void __launch_bounds__(CGM_RB) k_cgm_resolve(const int *__restrict__ order, long long n_own, const long long *__restrict__ off,
                                                       const int *__restrict__ nbr, unsigned char *state,
                                                       unsigned long long *__restrict__ undecided) {
    volatile unsigned char *vs = state;
    const int lane = threadIdx.x & 31;
    const long long warp = ((long long)blockIdx.x * CGM_RB + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * CGM_RB) >> 5;
    unsigned long long left = 0;
    for (long long b = warp * 32; b < n_own; b += nwarps * 32) {
        const long long k = b + lane;
        const int r = k < n_own ? order[k] : -1;
        bool pending = r >= 0 && vs[r] == CGM_UNDECIDED;
        while (true) {
            bool moved = false;
            if (pending) {
                bool sat = false, all_final = true;
                for (long long e = off[r], e1 = off[r + 1]; e < e1; e++) {
                    const unsigned char s = vs[nbr[e]];
                    if (s == CGM_CENTRAL) { sat = true; break; }
                    if (s == CGM_UNDECIDED) all_final = false;
                }
                if (sat || all_final) {
                    vs[r] = sat ? CGM_SATELLITE : CGM_CENTRAL;
                    pending = false;
                    moved = true;
                }
            }
            __threadfence_block();
            if (!__any_sync(0xffffffffu, moved)) break;
        }
        left += pending ? 1 : 0;
    }
    for (int o = 16; o > 0; o >>= 1) left += __shfl_down_sync(0xffffffffu, left, o);
    if (lane == 0 && left) atomicAdd(undecided, left);
}

// per owned satellite: the priority of its central (the highest-priority central among its higher-priority neighbours),
// and +1 on that central's satellite count; per owned central: its own priority
__global__ void __launch_bounds__(CGM_RB) k_cgm_assign(const int *__restrict__ order, long long n_own, const long long *__restrict__ off,
                                                      const int *__restrict__ nbr, const unsigned char *__restrict__ state,
                                                      const long long *__restrict__ sprio, long long *__restrict__ cen_prio,
                                                      unsigned long long *__restrict__ nsat) {
    const long long stride = (long long)gridDim.x * CGM_RB;
    for (long long k = (long long)blockIdx.x * CGM_RB + threadIdx.x; k < n_own; k += stride) {
        const int r = order[k];
        if (state[r] == CGM_CENTRAL) { cen_prio[r] = sprio[r]; continue; }
        long long bp = -1;
        int best = -1;
        for (long long e = off[r], e1 = off[r + 1]; e < e1; e++) {
            const int j = nbr[e];
            if (state[j] == CGM_CENTRAL && sprio[j] > bp) { bp = sprio[j]; best = j; }
        }
        cen_prio[r] = bp;
        if (best >= 0) atomicAdd(&nsat[best], 1ull);
    }
}

static int cgm_geom(PcGeom &g, CgmLink &lk, int periodic, const double *box_host, const int64_t *ncell_host, const double *tol_host,
                    const double *los_host, double rperp, double rpar) {
    NBK_CHECK_ARG(box_host != nullptr && ncell_host != nullptr && tol_host != nullptr, "cgm: box, cell counts and tolerances are required");
    NBK_CHECK_ARG(isfinite(rperp) && rperp >= 0 && isfinite(rpar) && rpar >= 0 && (rperp > 0 || rpar > 0),
                  "cgm: rperp and rpar must be finite, non-negative and not both 0 (got %g, %g)", rperp, rpar);
    if (los_host != nullptr)
        for (int d = 0; d < 3; d++) NBK_CHECK_ARG(isfinite(los_host[d]), "cgm: the line of sight must be finite");
    g = PcGeom{};
    g.periodic = periodic ? 1 : 0;
    lk.rperp2 = rperp * rperp;
    lk.rpar2 = rpar * rpar;
    const double rmax = sqrt(lk.rperp2 + lk.rpar2);
    // cells are skipped only when their nearest point is beyond rmax by a relative margin far above rounding
    g.thr_sph = lk.rperp2 + lk.rpar2;
    g.thr_sph = g.thr_sph * (1.0 + 1e-9) * (1.0 + 1e-9);
    g.thr_xy = g.thr_sph;
    double cells = 1.0;
    for (int d = 0; d < 3; d++) {
        NBK_CHECK_ARG(isfinite(box_host[d]) && box_host[d] > 0, "cgm: box side %d must be positive and finite", d);
        NBK_CHECK_ARG(ncell_host[d] >= 1 && ncell_host[d] <= CGM_MAX_CELLS_PER_AXIS, "cgm: cell count %lld on axis %d out of range",
                      (long long)ncell_host[d], d);
        NBK_CHECK_ARG(isfinite(tol_host[d]) && tol_host[d] >= 0, "cgm: bad tolerance on axis %d", d);
        g.box[d] = box_host[d];
        g.nc[d] = ncell_host[d];
        g.cs[d] = box_host[d] / (double)ncell_host[d];
        g.tol[d] = tol_host[d];
        const double reach = floor((rmax * (1.0 + 1e-9) + 2.0 * g.tol[d]) / g.cs[d] * (1.0 + 1e-12)) + 1.0;
        g.reach[d] = reach < (double)ncell_host[d] ? (long long)reach : (long long)ncell_host[d];
        lk.los[d] = los_host != nullptr ? los_host[d] : 0.0;
        cells *= (double)ncell_host[d];
    }
    NBK_CHECK_ARG(cells < 9.2e18, "cgm: %g cells do not fit a 63-bit key", cells);
    return NBK_OK;
}

static int cgm_walk(bool write, const double *spos, const int64_t *sprio, const uint32_t *perm, int64_t n, int64_t n_own,
                    const int64_t *chunk_first, const int64_t *chunk_key, int64_t nchunks, const uint32_t *cell_start,
                    const int64_t *cell_key, int64_t ncells, int periodic, const double *box_host, const int64_t *ncell_host,
                    const double *tol_host, const double *los_host, double rperp, double rpar, int64_t *counts,
                    const int64_t *offsets, int32_t *nbr, uint64_t *candidates, void *stream) {
    NBK_CHECK_ARG(n >= 0 && n < (1ll << 31), "cgm: %lld rows out of range (at most 2^31 - 1)", (long long)n);
    NBK_CHECK_ARG(n_own >= 0 && n_own <= n, "cgm: %lld owned rows of %lld", (long long)n_own, (long long)n);
    NBK_CHECK_ARG(nchunks >= 0 && nchunks < (1ll << 31), "cgm: chunk count %lld out of range", (long long)nchunks);
    NBK_CHECK_ARG(ncells >= 0 && ncells <= n, "cgm: cell count %lld out of range", (long long)ncells);
    PcGeom g;
    CgmLink lk;
    int rc = cgm_geom(g, lk, periodic, box_host, ncell_host, tol_host, los_host, rperp, rpar);
    if (rc) return rc;
    if (nchunks == 0 || ncells == 0 || n_own == 0) return NBK_OK;
    NBK_CHECK_ARG(spos && sprio && perm && chunk_first && chunk_key && cell_start && cell_key, "cgm: null device array");
    NBK_CHECK_ARG(write ? (offsets && nbr) : (counts && candidates), "cgm: null output array");
    cudaStream_t s = (cudaStream_t)stream;
    const long long *sp = (const long long *)sprio, *cf = (const long long *)chunk_first, *ck = (const long long *)chunk_key,
                    *sck = (const long long *)cell_key, *of = (const long long *)offsets;
    const unsigned *pm = (const unsigned *)perm, *cs = (const unsigned *)cell_start;
    long long *ct = (long long *)counts;
    unsigned long long *cd = (unsigned long long *)candidates;
    const bool flat = los_host != nullptr;
#define CGM_GO(W, F) k_cgm_walk<W, F><<<(unsigned)nchunks, CGM_B, 0, s>>>(spos, sp, pm, n_own, cf, ck, cs, sck, ncells, g, lk, ct, of, nbr, cd)
    if (write) { if (flat) CGM_GO(true, true); else CGM_GO(true, false); }
    else { if (flat) CGM_GO(false, true); else CGM_GO(false, false); }
#undef CGM_GO
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int64_t nbk_cgm_chunk_rows(void) { return CGM_B; }

extern "C" int nbk_cgm_count(const double *spos, const int64_t *sprio, const uint32_t *perm, int64_t n, int64_t n_own,
                             const int64_t *chunk_first, const int64_t *chunk_key, int64_t nchunks, const uint32_t *cell_start,
                             const int64_t *cell_key, int64_t ncells, int periodic, const double *box_host, const int64_t *ncell_host,
                             const double *tol_host, const double *los_host, double rperp, double rpar, int64_t *counts,
                             uint64_t *candidates, void *stream) {
    return cgm_walk(false, spos, sprio, perm, n, n_own, chunk_first, chunk_key, nchunks, cell_start, cell_key, ncells, periodic,
                    box_host, ncell_host, tol_host, los_host, rperp, rpar, counts, nullptr, nullptr, candidates, stream);
}

extern "C" int nbk_cgm_write(const double *spos, const int64_t *sprio, const uint32_t *perm, int64_t n, int64_t n_own,
                             const int64_t *chunk_first, const int64_t *chunk_key, int64_t nchunks, const uint32_t *cell_start,
                             const int64_t *cell_key, int64_t ncells, int periodic, const double *box_host, const int64_t *ncell_host,
                             const double *tol_host, const double *los_host, double rperp, double rpar, const int64_t *offsets,
                             int32_t *nbr, void *stream) {
    return cgm_walk(true, spos, sprio, perm, n, n_own, chunk_first, chunk_key, nchunks, cell_start, cell_key, ncells, periodic,
                    box_host, ncell_host, tol_host, los_host, rperp, rpar, nullptr, offsets, nbr, nullptr, stream);
}

extern "C" int nbk_cgm_resolve(const int32_t *order, int64_t n_own, const int64_t *offsets, const int32_t *nbr, uint8_t *state,
                               uint64_t *undecided, void *stream) {
    NBK_CHECK_ARG(n_own >= 0 && n_own < (1ll << 31), "cgm_resolve: %lld rows out of range", (long long)n_own);
    if (n_own == 0) return NBK_OK;
    NBK_CHECK_ARG(order && offsets && nbr && state && undecided, "cgm_resolve: null device array");
    cudaStream_t s = (cudaStream_t)stream;
    k_cgm_resolve<<<nbk_grid_for(n_own, CGM_RB, 8), CGM_RB, 0, s>>>(order, n_own, (const long long *)offsets, nbr, state,
                                                                    (unsigned long long *)undecided);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_cgm_assign(const int32_t *order, int64_t n_own, const int64_t *offsets, const int32_t *nbr, const uint8_t *state,
                              const int64_t *sprio, int64_t *cen_prio, uint64_t *nsat, void *stream) {
    NBK_CHECK_ARG(n_own >= 0 && n_own < (1ll << 31), "cgm_assign: %lld rows out of range", (long long)n_own);
    if (n_own == 0) return NBK_OK;
    NBK_CHECK_ARG(order && offsets && nbr && state && sprio && cen_prio && nsat, "cgm_assign: null device array");
    cudaStream_t s = (cudaStream_t)stream;
    k_cgm_assign<<<nbk_grid_for(n_own, CGM_RB, 8), CGM_RB, 0, s>>>(order, n_own, (const long long *)offsets, nbr, state,
                                                                   (const long long *)sprio, (long long *)cen_prio,
                                                                   (unsigned long long *)nsat);
    NBK_LAUNCHED();
    return NBK_OK;
}
