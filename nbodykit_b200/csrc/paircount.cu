// Binned pair counts in a simulation box (nbodykit/algorithms/pair_counters/simbox.py: the Corrfunc DD / DDsmu / DDrppi
// calls of SimulationBoxPairCount) on the cell grid of csrc/fof.cu.
//   nbk_paircount : for every primary row (sorted by cell key, split into chunks of at most PC_B rows of one cell) and
//                   every secondary row in a cell within reach, add the ordered pair to its bin: npairs (uint64),
//                   sum of w1 * w2 and sum of the separation (s, or r_p in 'projected'), all in double.
// One CTA per chunk: the primaries sit in registers, the secondaries of each neighbour column (a contiguous range of
// key-sorted rows) are staged through shared memory in tiles of PC_B rows, and every thread tests the whole tile
// against its primary.  The histogram lives in shared memory when it fits (PC_SMEM_BINS) and is flushed once per CTA
// with 64-bit integer and f64 atomics; larger histograms take global atomics directly.
// Separations: |d| per axis in double from the wrapped positions (periodic: min(|d|, L - |d|)), r_p^2 = da^2 + db^2,
// s^2 = r_p^2 + dc^2 with c the line of sight (the last column).  The file is compiled with --fmad=false: no
// contraction may move a pair across a bin edge.
#include "pc_cells.cuh"

#include <math.h>

#define PC_B 128
#define PC_SMEM_BINS 1024
#define PC_MAX_EDGES 4097
#define PC_MAX_CELLS_PER_AXIS (1ll << 21)

// largest k in [0, n) with e[k] <= v, given e[0] <= v (right-open bins; v beyond e[n] lands in bin n - 1)
static __device__ __forceinline__ int pc_bin(const double *e, int n, double v) {
    int lo = 0, hi = n;
    while (hi - lo > 1) {
        int mid = (lo + hi) >> 1;
        if (e[mid] <= v) lo = mid; else hi = mid;
    }
    return lo;
}

template <bool SMEM>
static __device__ __forceinline__ void pc_add(int b, double ww, double sep, unsigned long long *cnt, double *wsum, double *ssum) {
    atomicAdd(&cnt[b], 1ull);
    atomicAdd(&wsum[b], ww);
    atomicAdd(&ssum[b], sep);
}

template <int MODE, bool SMEM>
__global__ void __launch_bounds__(PC_B, 4) k_paircount(const double *__restrict__ ppos, const double *__restrict__ pw,
                                                    const long long *__restrict__ chunk_first, const long long *__restrict__ chunk_key,
                                                    const double *__restrict__ spos, const double *__restrict__ sw,
                                                    const unsigned *__restrict__ scell_start, const long long *__restrict__ scell_key,
                                                    int64_t nscells, PcGeom g, const double *__restrict__ e2_g,
                                                    const double *__restrict__ e2nd_g, unsigned long long *__restrict__ g_cnt,
                                                    double *__restrict__ g_wsum, double *__restrict__ g_ssum,
                                                    unsigned long long *__restrict__ g_cand) {
    extern __shared__ double sm[];
    double *tile = sm;                                  // [4][PC_B]: x, y, z, w
    double *e2 = tile + 4 * PC_B;                       // nb + 1 squared edges
    double *e2nd = e2 + (g.nb + 1);                     // n2 + 1 mu / pi edges
    const int nbins = g.nb * g.n2;
    unsigned long long *cnt = g_cnt;
    double *wsum = g_wsum, *ssum = g_ssum;
    if (SMEM) {
        cnt = (unsigned long long *)(e2nd + (g.n2 + 1));
        wsum = (double *)(cnt + nbins);
        ssum = wsum + nbins;
        for (int b = threadIdx.x; b < nbins; b += PC_B) { cnt[b] = 0ull; wsum[b] = 0.0; ssum[b] = 0.0; }
    }
    for (int k = threadIdx.x; k <= g.nb; k += PC_B) e2[k] = e2_g[k];
    if (MODE != NBK_PC_1D && MODE != NBK_PC_ANGULAR)
        for (int k = threadIdx.x; k <= g.n2; k += PC_B) e2nd[k] = e2nd_g[k];

    const int64_t c = blockIdx.x;
    const long long p0 = chunk_first[c], np = chunk_first[c + 1] - p0;
    const long long key = chunk_key[c];
    const long long nyz = g.nc[1] * g.nc[2];
    const long long ix = key / nyz, iy = (key / g.nc[2]) % g.nc[1], iz = key % g.nc[2];
    const bool have = threadIdx.x < np;
    double px = 0.0, py = 0.0, pz = 0.0, pwt = 0.0;
    if (have) {
        const long long r = p0 + threadIdx.x;
        px = ppos[3 * r]; py = ppos[3 * r + 1]; pz = ppos[3 * r + 2]; pwt = pw[r];
    }
    __syncthreads();
    const double emin2 = e2[0], emax2 = e2[g.nb];
    unsigned long long cand = 0;

    const PcAxis ax = pc_axis(ix, g.reach[0], 0, g), ay = pc_axis(iy, g.reach[1], 1, g);
    for (long long xx = ax.lo; xx <= ax.hi; xx++) {
        const long long x = g.periodic ? pc_wrap(xx, g.nc[0]) : xx;
        const double gx = axis_gap(pc_delta(xx, ix, ax.all, g.nc[0]), 0, g);
        for (long long yy = ay.lo; yy <= ay.hi; yy++) {
            const long long y = g.periodic ? pc_wrap(yy, g.nc[1]) : yy;
            const double gy = axis_gap(pc_delta(yy, iy, ay.all, g.nc[1]), 1, g);
            const double gxy2 = gx * gx + gy * gy;
            if (gxy2 >= g.thr_xy) continue;
            // the z cells this column can still reach: gap_z < rem
            double rem = MODE == NBK_PC_PROJECTED ? g.pimax : sqrt(g.thr_sph - gxy2);
            double rzd = floor((rem + g.tol[2]) / g.cs[2]) + 1.0;
            long long rz = rzd < (double)g.reach[2] ? (long long)rzd : g.reach[2];
            const PcAxis az = pc_axis(iz, rz, 2, g);
            long long z0[2], z1[2];
            int nr = 0;
            if (az.all || !g.periodic) { z0[nr] = az.lo; z1[nr++] = az.hi; }
            else if (az.lo < 0) { z0[nr] = az.lo + g.nc[2]; z1[nr++] = g.nc[2] - 1; z0[nr] = 0; z1[nr++] = az.hi; }
            else if (az.hi >= g.nc[2]) { z0[nr] = az.lo; z1[nr++] = g.nc[2] - 1; z0[nr] = 0; z1[nr++] = az.hi - g.nc[2]; }
            else { z0[nr] = az.lo; z1[nr++] = az.hi; }
            const long long row = (x * g.nc[1] + y) * g.nc[2];
            for (int q = 0; q < nr; q++) {
                // the occupied cells of keys row + [z0, z1] are consecutive, and so are their key-sorted rows
                const int64_t d0 = pc_lower_bound(scell_key, nscells, row + z0[q]);
                const int64_t d1 = pc_lower_bound(scell_key, nscells, row + z1[q] + 1);
                if (d0 >= d1) continue;
                const long long r0 = scell_start[d0], r1 = scell_start[d1];
                for (long long base = r0; base < r1; base += PC_B) {
                    const int m = (int)(r1 - base < PC_B ? r1 - base : PC_B);
                    __syncthreads();
                    if (threadIdx.x < m) {
                        const long long r = base + threadIdx.x;
                        tile[threadIdx.x] = spos[3 * r];
                        tile[PC_B + threadIdx.x] = spos[3 * r + 1];
                        tile[2 * PC_B + threadIdx.x] = spos[3 * r + 2];
                        tile[3 * PC_B + threadIdx.x] = sw[r];
                    }
                    __syncthreads();
                    cand += (unsigned long long)m;
                    if (!have) continue;
                    for (int j = 0; j < m; j++) {
                        double da = fabs(px - tile[j]), db = fabs(py - tile[PC_B + j]), dc = fabs(pz - tile[2 * PC_B + j]);
                        if (g.periodic) {
                            da = fmin(da, g.box[0] - da);
                            db = fmin(db, g.box[1] - db);
                            dc = fmin(dc, g.box[2] - dc);
                        }
                        const double rp2 = da * da + db * db;
                        if (MODE == NBK_PC_SURVEY_2D || MODE == NBK_PC_SURVEY_PROJECTED) {
                            // the line of sight of the pair is its midpoint: l = x1 + x2, observer at the origin
                            const double s2 = rp2 + dc * dc;
                            if (MODE == NBK_PC_SURVEY_2D ? (s2 < emin2 || !(s2 < emax2)) : !(s2 < g.thr_sph)) continue;
                            const double sx = tile[j] - px, sy = tile[PC_B + j] - py, sz = tile[2 * PC_B + j] - pz;
                            const double lx = px + tile[j], ly = py + tile[PC_B + j], lz = pz + tile[2 * PC_B + j];
                            const double l2 = (lx * lx + ly * ly) + lz * lz;
                            const double sl = (sx * lx + sy * ly) + sz * lz;
                            if (MODE == NBK_PC_SURVEY_2D) {
                                const double s = sqrt(s2);
                                const double mu = l2 > 0.0 ? fabs(sl) / (s * sqrt(l2)) : 0.0;
                                const int b = pc_bin(e2, g.nb, s2) * g.n2 + pc_bin(e2nd, g.n2, mu);
                                pc_add<SMEM>(b, pwt * tile[3 * PC_B + j], s, cnt, wsum, ssum);
                            } else {
                                const double pi = l2 > 0.0 ? fabs(sl) / sqrt(l2) : 0.0;
                                if (!(pi < g.pimax)) continue;
                                double rq2 = s2 - pi * pi;
                                rq2 = rq2 > 0.0 ? rq2 : 0.0;
                                if (rq2 < emin2 || !(rq2 < emax2)) continue;
                                const int b = pc_bin(e2, g.nb, rq2) * g.n2 + pc_bin(e2nd, g.n2, pi);
                                pc_add<SMEM>(b, pwt * tile[3 * PC_B + j], sqrt(rq2), cnt, wsum, ssum);
                            }
                        } else if (MODE == NBK_PC_ANGULAR) {
                            // unit vectors: bins of the chord, summed as the angle in degrees
                            const double s2 = rp2 + dc * dc;
                            if (s2 < emin2 || !(s2 < emax2)) continue;
                            const double theta = 2.0 * asin(0.5 * sqrt(s2)) * (180.0 / M_PI);
                            pc_add<SMEM>(pc_bin(e2, g.nb, s2), pwt * tile[3 * PC_B + j], theta, cnt, wsum, ssum);
                        } else if (MODE == NBK_PC_PROJECTED) {
                            if (!(dc < g.pimax) || rp2 < emin2 || !(rp2 < emax2)) continue;
                            const int b = pc_bin(e2, g.nb, rp2) * g.n2 + pc_bin(e2nd, g.n2, dc);
                            pc_add<SMEM>(b, pwt * tile[3 * PC_B + j], sqrt(rp2), cnt, wsum, ssum);
                        } else {
                            const double s2 = rp2 + dc * dc;
                            if (s2 < emin2 || !(s2 < emax2)) continue;
                            const double s = sqrt(s2);
                            int b = pc_bin(e2, g.nb, s2);
                            if (MODE == NBK_PC_2D) b = b * g.n2 + pc_bin(e2nd, g.n2, dc / s);
                            pc_add<SMEM>(b, pwt * tile[3 * PC_B + j], s, cnt, wsum, ssum);
                        }
                    }
                }
            }
        }
    }
    if (threadIdx.x == 0) atomicAdd(g_cand, cand * (unsigned long long)np);
    if (SMEM) {
        __syncthreads();
        for (int b = threadIdx.x; b < nbins; b += PC_B) {
            if (cnt[b]) {
                atomicAdd(&g_cnt[b], cnt[b]);
                atomicAdd(&g_wsum[b], wsum[b]);
                atomicAdd(&g_ssum[b], ssum[b]);
            }
        }
    }
}

template <int MODE, bool SMEM>
static int pc_launch(int64_t nchunks, size_t shm, cudaStream_t s, const double *ppos, const double *pw, const long long *chunk_first,
                     const long long *chunk_key, const double *spos, const double *sw, const unsigned *scs, const long long *sck,
                     int64_t nscells, const PcGeom &g, const double *e2, const double *e2nd, unsigned long long *cnt, double *wsum,
                     double *ssum, unsigned long long *cand) {
    auto kern = k_paircount<MODE, SMEM>;
    if (shm > 48 * 1024) NBK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
    kern<<<(unsigned)nchunks, PC_B, shm, s>>>(ppos, pw, chunk_first, chunk_key, spos, sw, scs, sck, nscells, g, e2, e2nd, cnt, wsum, ssum,
                                              cand);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int64_t nbk_paircount_chunk_rows(void) { return PC_B; }
extern "C" int64_t nbk_paircount_smem_bins(void) { return PC_SMEM_BINS; }

extern "C" int nbk_paircount(int mode, const double *ppos, const double *pw, const int64_t *chunk_first, const int64_t *chunk_key,
                             int64_t nchunks, const double *spos, const double *sw, const uint32_t *scell_start,
                             const int64_t *scell_key, int64_t nscells, int periodic, const double *box_host,
                             const int64_t *ncell_host, const double *tol_host, const double *edges_host, int nedges,
                             const double *edges2_host, int nedges2, double pimax, double *work, uint64_t *npairs, double *wsum,
                             double *ssum, uint64_t *candidates, void *stream) {
    NBK_CHECK_ARG(mode >= NBK_PC_1D && mode <= NBK_PC_ANGULAR, "paircount: bad mode %d", mode);
    const bool survey = mode >= NBK_PC_SURVEY_2D;
    const bool projected = mode == NBK_PC_PROJECTED || mode == NBK_PC_SURVEY_PROJECTED;
    const bool one_dim = mode == NBK_PC_1D || mode == NBK_PC_ANGULAR;
    NBK_CHECK_ARG(!(survey && periodic), "paircount: mode %d (survey / angular) is not periodic", mode);
    NBK_CHECK_ARG(nchunks >= 0 && nchunks < (1ll << 31), "paircount: chunk count %lld out of range", (long long)nchunks);
    NBK_CHECK_ARG(nscells >= 0 && nscells < (1ll << 32), "paircount: cell count %lld out of range", (long long)nscells);
    NBK_CHECK_ARG(box_host != nullptr && ncell_host != nullptr && tol_host != nullptr && edges_host != nullptr,
                  "paircount: box, cell counts, tolerances and edges are required");
    NBK_CHECK_ARG(nedges >= 2 && nedges <= PC_MAX_EDGES, "paircount: %d edges (2 .. %d supported)", nedges, PC_MAX_EDGES);
    for (int k = 0; k < nedges; k++) {
        NBK_CHECK_ARG(isfinite(edges_host[k]) && edges_host[k] > 0, "paircount: edges must be positive and finite");
        NBK_CHECK_ARG(k == 0 || edges_host[k] > edges_host[k - 1], "paircount: edges must increase strictly");
    }
    PcGeom g;
    g.mode = mode;
    g.periodic = periodic ? 1 : 0;
    g.nb = nedges - 1;
    g.n2 = 1;
    if (!one_dim) {
        NBK_CHECK_ARG(edges2_host != nullptr && nedges2 >= 2 && nedges2 <= PC_MAX_EDGES,
                      "paircount: %d second-dimension edges (2 .. %d supported)", nedges2, PC_MAX_EDGES);
        g.n2 = nedges2 - 1;
    }
    NBK_CHECK_ARG((int64_t)g.nb * g.n2 < (1ll << 31), "paircount: too many bins");
    const double emax = edges_host[nedges - 1];
    double smax2 = emax * emax;
    g.pimax = 0.0;
    if (projected) {
        NBK_CHECK_ARG(isfinite(pimax) && pimax > 0, "paircount: pimax must be positive and finite (got %g)", pimax);
        g.pimax = pimax;
        smax2 = smax2 + pimax * pimax;
    }
    // the skip thresholds: a relative margin far above the rounding of the gaps and of the pair separations.  A survey
    // pair's line of sight is its own, so survey 'projected' prunes on the sphere s_max^2 = r_p,max^2 + pimax^2.
    g.thr_xy = (mode == NBK_PC_PROJECTED ? emax * emax : smax2) * (1.0 + 1e-9);
    g.thr_sph = smax2 * (1.0 + 1e-9);
    const double smax = sqrt(smax2);
    double cells = 1.0;
    for (int d = 0; d < 3; d++) {
        NBK_CHECK_ARG(isfinite(box_host[d]) && box_host[d] > 0, "paircount: box side %d must be positive and finite", d);
        NBK_CHECK_ARG(ncell_host[d] >= 1 && ncell_host[d] <= PC_MAX_CELLS_PER_AXIS, "paircount: cell count %lld on axis %d out of range",
                      (long long)ncell_host[d], d);
        NBK_CHECK_ARG(isfinite(tol_host[d]) && tol_host[d] >= 0, "paircount: bad tolerance on axis %d", d);
        g.box[d] = box_host[d];
        g.nc[d] = ncell_host[d];
        g.cs[d] = box_host[d] / (double)ncell_host[d];
        g.tol[d] = tol_host[d];
        g.reach[d] = (long long)floor((smax + 2.0 * g.tol[d]) / g.cs[d] * (1.0 + 1e-12)) + 1;
        cells *= (double)ncell_host[d];
    }
    NBK_CHECK_ARG(cells < 9.2e18, "paircount: %g cells do not fit a 63-bit key", cells);
    const int nbins = g.nb * g.n2;
    const bool smem = nbins <= PC_SMEM_BINS;
    size_t shm = sizeof(double) * (4 * PC_B + (g.nb + 1) + (g.n2 + 1)) + (smem ? (size_t)nbins * 24 : 0);
    if (nchunks == 0 || nscells == 0) return NBK_OK;
    NBK_CHECK_ARG(work != nullptr, "paircount: a device workspace of %d doubles is required", (g.nb + 1) + (g.n2 + 1));
    cudaStream_t s = (cudaStream_t)stream;
    // squared edges (host, double) and the mu / pi edges as given, staged once through the workspace
    double *hbuf = (double *)malloc(sizeof(double) * ((g.nb + 1) + (g.n2 + 1)));
    NBK_CHECK_ARG(hbuf != nullptr, "paircount: out of host memory");
    for (int k = 0; k <= g.nb; k++) hbuf[k] = edges_host[k] * edges_host[k];
    for (int k = 0; k <= g.n2; k++) hbuf[g.nb + 1 + k] = one_dim ? 0.0 : edges2_host[k];
    cudaError_t e = cudaMemcpyAsync(work, hbuf, sizeof(double) * ((g.nb + 1) + (g.n2 + 1)), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    free(hbuf);
    NBK_CUDA(e);
    const double *e2 = work, *e2nd = work + (g.nb + 1);
    const long long *cf = (const long long *)chunk_first, *ck = (const long long *)chunk_key, *sck = (const long long *)scell_key;
    const unsigned *scs = (const unsigned *)scell_start;
    unsigned long long *cnt = (unsigned long long *)npairs, *cand = (unsigned long long *)candidates;
#define PC_GO(M, S) pc_launch<M, S>(nchunks, shm, s, ppos, pw, cf, ck, spos, sw, scs, sck, nscells, g, e2, e2nd, cnt, wsum, ssum, cand)
    if (mode == NBK_PC_1D) return smem ? PC_GO(NBK_PC_1D, true) : PC_GO(NBK_PC_1D, false);
    if (mode == NBK_PC_2D) return smem ? PC_GO(NBK_PC_2D, true) : PC_GO(NBK_PC_2D, false);
    if (mode == NBK_PC_PROJECTED) return smem ? PC_GO(NBK_PC_PROJECTED, true) : PC_GO(NBK_PC_PROJECTED, false);
    if (mode == NBK_PC_SURVEY_2D) return smem ? PC_GO(NBK_PC_SURVEY_2D, true) : PC_GO(NBK_PC_SURVEY_2D, false);
    if (mode == NBK_PC_SURVEY_PROJECTED)
        return smem ? PC_GO(NBK_PC_SURVEY_PROJECTED, true) : PC_GO(NBK_PC_SURVEY_PROJECTED, false);
    return smem ? PC_GO(NBK_PC_ANGULAR, true) : PC_GO(NBK_PC_ANGULAR, false);
#undef PC_GO
}
