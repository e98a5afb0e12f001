// Multipoles of the isotropic three-point correlation function in a simulation box (nbodykit/algorithms/threeptcf.py:
// SimulationBox3PCF) on the cell grid of csrc/fof.cu, with the neighbour walk of csrc/paircount.cu (pc_cells.cuh).
//   nbk_threeptcf : zeta_l(b1, b2) += sum_p w_p sum_m c_m Re[a_lm(b1) a*_lm(b2)] for b1 <= b2 (c_0 = 1, c_m>0 = 2),
//                   with a_lm(b) = sum_{j in b} w_j Y_lm(u_pj) up to the constant 1 / (16 pi^2) applied by the caller.
// Y_lm(u) is proportional to (ux + i uy)^m Q_lm(uz) with Q_lm a polynomial of degree l - m, so per primary and radial
// bin the kernel accumulates the complex moments M_{m,k}(b) = sum_j w_j (ux + i uy)^m uz^k (m + k <= lmax) and turns
// them into a_lm = sum_k T_lmk M_{m,k} with the host-built table T (exact rationals times the normalisation, rounded
// once to double).
// One CTA per chunk of at most TP_CHUNK primaries of one cell; each of its NW warps takes one primary per round.  The
// secondaries of each neighbour column are staged through shared memory for all warps; a warp's lanes take one
// neighbour each (separation, bin, power ladders into per-warp scratch), then one moment each, accumulating into the
// warp's [nb][nmom] moments in shared memory (each lane owns its addresses: no atomics).  At the end of a round every
// thread of the CTA owns some (l, b1, b2) entries of the CTA's zeta and adds the round's primaries into them; zeta and
// the per-bin pair counts are flushed once per CTA with global atomics.
// Separations: d = x_j - x_p per axis in double (periodic: d > L/2 -> d - L, d <= -L/2 -> d + L), r = sqrt((dx^2 +
// dy^2) + dz^2); bin k holds e_k < r <= e_{k+1} and r > 0.  The file is compiled with --fmad=false so that no
// contraction can move a pair across a bin edge; the moment and zeta sums use explicit fma().
#include "pc_cells.cuh"

#include <math.h>

#define TP_CHUNK 128
#define TP_MAX_L 10
#define TP_MAX_POLES (TP_MAX_L + 1)
#define TP_MAX_NB 32
#define TP_MAX_NW 8
#define TP_MAX_CELLS_PER_AXIS (1ll << 21)

struct TpParam {
    int L;       // largest pole
    int nmom;    // (L + 1) (L + 2) / 2 moments M_{m,k}, m + k <= L; also the number of a_lm, 0 <= m <= l <= L
    int npole;   // requested poles
    int nb;      // radial bins
    int nbp;     // bin pairs b1 <= b2
    int nw;      // warps per CTA
    int poles[TP_MAX_POLES];
};

// moments and harmonics share one layout: m-major, offset(m) = sum_{m' < m} (L + 1 - m'); M_{m,k} at offset(m) + k,
// a_lm at offset(m) + (l - m)
static __device__ __forceinline__ int tp_off(int m, int L) { return m * (L + 1) - (m * (m - 1)) / 2; }

__global__ void __launch_bounds__(32 * TP_MAX_NW) k_threeptcf(
        const double *__restrict__ ppos, const double *__restrict__ pw, const long long *__restrict__ chunk_first,
        const long long *__restrict__ chunk_key, const double *__restrict__ spos, const double *__restrict__ sw,
        const unsigned *__restrict__ scell_start, const long long *__restrict__ scell_key, int64_t nscells, PcGeom g,
        TpParam t, const double *__restrict__ edges_g, const double *__restrict__ coef, double *__restrict__ g_zeta,
        unsigned long long *__restrict__ g_npairs, unsigned long long *__restrict__ g_cand) {
    extern __shared__ double sm[];
    const int NT = blockDim.x, L1 = t.L + 1, nmom = t.nmom, nb = t.nb;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nz = t.npole * t.nbp;
    // shared layout (doubles first, then 8-byte counters, then ints)
    double *tile = sm;                                   // [4][NT]: x, y, z, w
    double *edges = tile + 4 * NT;                       // nb + 1
    double *zeta = edges + (nb + 1);                     // [npole][nbp]
    double *pwt = zeta + nz;                             // [nw] primary weight of the round (0: no primary)
    double *acc = pwt + t.nw;                            // [nw][nb][nmom][2]
    double *scr = acc + (size_t)t.nw * nb * nmom * 2;    // [nw][3][32][L + 1]: Re, Im of (ux + i uy)^m, w uz^k
    unsigned long long *cnt = (unsigned long long *)(scr + (size_t)t.nw * 3 * 32 * L1);   // [nb]
    int *sbin = (int *)(cnt + nb);                       // [nw][32]
    int *pairs = sbin + t.nw * 32;                       // [nbp]: b1 << 8 | b2

    for (int k = threadIdx.x; k <= nb; k += NT) edges[k] = edges_g[k];
    for (int k = threadIdx.x; k < nz; k += NT) zeta[k] = 0.0;
    for (int k = threadIdx.x; k < nb; k += NT) cnt[k] = 0ull;
    for (int k = threadIdx.x; k < t.nbp; k += NT) {
        int b1 = 0, r = k;
        while (r >= nb - b1) { r -= nb - b1; b1++; }
        pairs[k] = (b1 << 8) | (b1 + r);
    }
    double *wacc = acc + (size_t)warp * nb * nmom * 2;
    double *xr = scr + (size_t)warp * 3 * 32 * L1, *xi = xr + 32 * L1, *wz = xi + 32 * L1;
    int *wbin = sbin + warp * 32;
    // the moments this lane owns: q = lane, lane + 32, lane + 64 (nmom <= 66)
    int qm[3], qk[3];
    for (int s = 0; s < 3; s++) {
        int q = lane + 32 * s, m = 0;
        qm[s] = -1; qk[s] = 0;
        if (q < nmom) {
            while (q >= L1 - m) { q -= L1 - m; m++; }
            qm[s] = m; qk[s] = q;
        }
    }

    const int64_t c = blockIdx.x;
    const long long p0 = chunk_first[c], np = chunk_first[c + 1] - p0;
    const long long key = chunk_key[c];
    const long long nyz = g.nc[1] * g.nc[2];
    const long long ix = key / nyz, iy = (key / g.nc[2]) % g.nc[1], iz = key % g.nc[2];
    const double h0 = 0.5 * g.box[0], h1 = 0.5 * g.box[1], h2 = 0.5 * g.box[2];
    unsigned long long cand = 0;
    __syncthreads();
    const double emin = edges[0], emax = edges[nb];

    for (long long round = 0; round * t.nw < np; round++) {
        const long long ip = round * t.nw + warp;
        const bool have = ip < np;
        double px = 0.0, py = 0.0, pz = 0.0;
        if (have) {
            const long long r = p0 + ip;
            px = ppos[3 * r]; py = ppos[3 * r + 1]; pz = ppos[3 * r + 2];
        }
        if (lane == 0) pwt[warp] = have ? pw[p0 + ip] : 0.0;
        for (int k = lane; k < nb * nmom * 2; k += 32) wacc[k] = 0.0;
        __syncwarp();

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
                double rem = sqrt(g.thr_sph - gxy2);
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
                    const int64_t d0 = pc_lower_bound(scell_key, nscells, row + z0[q]);
                    const int64_t d1 = pc_lower_bound(scell_key, nscells, row + z1[q] + 1);
                    if (d0 >= d1) continue;
                    const long long r0 = scell_start[d0], r1 = scell_start[d1];
                    for (long long base = r0; base < r1; base += NT) {
                        const int m = (int)(r1 - base < NT ? r1 - base : NT);
                        __syncthreads();
                        if (threadIdx.x < m) {
                            const long long r = base + threadIdx.x;
                            tile[threadIdx.x] = spos[3 * r];
                            tile[NT + threadIdx.x] = spos[3 * r + 1];
                            tile[2 * NT + threadIdx.x] = spos[3 * r + 2];
                            tile[3 * NT + threadIdx.x] = sw[r];
                        }
                        __syncthreads();
                        if (!have) continue;
                        if (lane == 0) cand += (unsigned long long)m;
                        for (int s0 = 0; s0 < m; s0 += 32) {
                            const int j = s0 + lane;
                            bool ok = false;
                            int b = 0;
                            double dx = 0.0, dy = 0.0, dz = 0.0, r = 0.0;
                            if (j < m) {
                                dx = tile[j] - px; dy = tile[NT + j] - py; dz = tile[2 * NT + j] - pz;
                                if (g.periodic) {
                                    if (dx > h0) dx -= g.box[0]; else if (dx <= -h0) dx += g.box[0];
                                    if (dy > h1) dy -= g.box[1]; else if (dy <= -h1) dy += g.box[1];
                                    if (dz > h2) dz -= g.box[2]; else if (dz <= -h2) dz += g.box[2];
                                }
                                r = sqrt((dx * dx + dy * dy) + dz * dz);
                                ok = r > 0.0 && r > emin && r <= emax;
                                if (ok) {
                                    // the largest k with e_k < r
                                    int lo = 0, hi = nb;
                                    while (hi - lo > 1) {
                                        const int mid = (lo + hi) >> 1;
                                        if (edges[mid] < r) lo = mid; else hi = mid;
                                    }
                                    b = lo;
                                }
                            }
                            const unsigned mask = __ballot_sync(0xffffffffu, ok);
                            if (mask == 0u) continue;
                            if (ok) {
                                const int slot = __popc(mask & ((1u << lane) - 1u));
                                const unsigned same = __match_any_sync(mask, b);
                                if (lane == __ffs(same) - 1) atomicAdd(&cnt[b], (unsigned long long)__popc(same));
                                wbin[slot] = b;
                                const double ux = dx / r, uy = dy / r, uz = dz / r;
                                double er = 1.0, ei = 0.0, zk = tile[3 * NT + j];
                                for (int k = 0; k < L1; k++) {
                                    xr[slot * L1 + k] = er; xi[slot * L1 + k] = ei; wz[slot * L1 + k] = zk;
                                    const double nr_ = er * ux - ei * uy;
                                    ei = er * uy + ei * ux;
                                    er = nr_;
                                    zk = zk * uz;
                                }
                            }
                            __syncwarp();
                            const int nok = __popc(mask);
                            // one moment per lane: runs of neighbours in one bin are summed in registers
                            for (int s = 0; s < 3; s++) {
                                if (qm[s] < 0) break;
                                const int mm = qm[s], kk = qk[s];
                                double ar = 0.0, ai = 0.0;
                                int cur = wbin[0];
                                for (int jj = 0; jj < nok; jj++) {
                                    const int bj = wbin[jj];
                                    if (bj != cur) {
                                        double *a = wacc + ((size_t)cur * nmom + (lane + 32 * s)) * 2;
                                        a[0] += ar; a[1] += ai;
                                        ar = 0.0; ai = 0.0; cur = bj;
                                    }
                                    const double z = wz[jj * L1 + kk];
                                    ar = fma(xr[jj * L1 + mm], z, ar);
                                    ai = fma(xi[jj * L1 + mm], z, ai);
                                }
                                double *a = wacc + ((size_t)cur * nmom + (lane + 32 * s)) * 2;
                                a[0] += ar; a[1] += ai;
                            }
                            __syncwarp();
                        }
                    }
                }
            }
        }
        // moments -> a_lm, in place per bin: a_lm at offset(m) + (l - m) needs M_{m,k} for k <= l - m of the same m
        if (have) {
            for (int b = 0; b < nb; b++) {
                double *row = wacc + (size_t)b * nmom * 2;
                double vr[3], vi[3];
                for (int s = 0; s < 3; s++) {
                    vr[s] = 0.0; vi[s] = 0.0;
                    if (qm[s] < 0) continue;
                    const int q = lane + 32 * s, o = tp_off(qm[s], t.L), jl = qk[s];   // l - m = jl
                    const double *cf = coef + (size_t)q * L1;
                    for (int k = jl & 1; k <= jl; k += 2) {
                        vr[s] = fma(cf[k], row[2 * (o + k)], vr[s]);
                        vi[s] = fma(cf[k], row[2 * (o + k) + 1], vi[s]);
                    }
                }
                __syncwarp();
                for (int s = 0; s < 3; s++) {
                    if (qm[s] < 0) continue;
                    row[2 * (lane + 32 * s)] = vr[s]; row[2 * (lane + 32 * s) + 1] = vi[s];
                }
                __syncwarp();
            }
        }
        __syncthreads();
        // this round's primaries into the CTA's zeta: each thread owns entries e = tid, tid + NT, ...
        for (int e = threadIdx.x; e < nz; e += NT) {
            const int pole = e / t.nbp, pr = pairs[e - pole * t.nbp];
            const int ell = t.poles[pole], b1 = pr >> 8, b2 = pr & 255;
            double z = zeta[e];
            for (int w = 0; w < t.nw; w++) {
                const double wp = pwt[w];
                if (wp == 0.0) continue;
                const double *a1 = acc + ((size_t)w * nb + b1) * nmom * 2, *a2 = acc + ((size_t)w * nb + b2) * nmom * 2;
                double s = 0.0;
                for (int m = 0; m <= ell; m++) {
                    const int i = 2 * (tp_off(m, t.L) + ell - m);
                    double v = fma(a1[i], a2[i], a1[i + 1] * a2[i + 1]);
                    s = fma(m == 0 ? 1.0 : 2.0, v, s);
                }
                z = fma(wp, s, z);
            }
            zeta[e] = z;
        }
        __syncthreads();
    }
    if (lane == 0 && cand) atomicAdd(g_cand, cand);
    for (int e = threadIdx.x; e < nz; e += NT) {
        const int pole = e / t.nbp, pr = pairs[e - pole * t.nbp];
        if (zeta[e] != 0.0) atomicAdd(&g_zeta[((size_t)pole * nb + (pr >> 8)) * nb + (pr & 255)], zeta[e]);
    }
    for (int k = threadIdx.x; k < nb; k += NT)
        if (cnt[k]) atomicAdd(&g_npairs[k], cnt[k]);
}

static size_t tp_smem(int nw, int nb, int nmom, int L, int npole) {
    const int nbp = nb * (nb + 1) / 2;
    return sizeof(double) * ((size_t)4 * 32 * nw + (nb + 1) + (size_t)npole * nbp + nw + (size_t)nw * nb * nmom * 2 +
                             (size_t)nw * 3 * 32 * (L + 1)) +
           sizeof(unsigned long long) * nb + sizeof(int) * ((size_t)nw * 32 + nbp);
}

extern "C" int64_t nbk_threeptcf_chunk_rows(void) { return TP_CHUNK; }
extern "C" int nbk_threeptcf_max_ell(void) { return TP_MAX_L; }
extern "C" int nbk_threeptcf_max_bins(void) { return TP_MAX_NB; }

extern "C" int nbk_threeptcf(const double *ppos, const double *pw, const int64_t *chunk_first, const int64_t *chunk_key,
                             int64_t nchunks, const double *spos, const double *sw, const uint32_t *scell_start,
                             const int64_t *scell_key, int64_t nscells, int periodic, const double *box_host,
                             const int64_t *ncell_host, const double *tol_host, const double *edges_host, int nedges,
                             const int *poles_host, int npoles, const double *coef_host, double *work, double *zeta,
                             uint64_t *npairs, uint64_t *candidates, void *stream) {
    NBK_CHECK_ARG(nchunks >= 0 && nchunks < (1ll << 31), "threeptcf: chunk count %lld out of range", (long long)nchunks);
    NBK_CHECK_ARG(nscells >= 0 && nscells < (1ll << 32), "threeptcf: cell count %lld out of range", (long long)nscells);
    NBK_CHECK_ARG(box_host != nullptr && ncell_host != nullptr && tol_host != nullptr && edges_host != nullptr &&
                      poles_host != nullptr && coef_host != nullptr,
                  "threeptcf: box, cell counts, tolerances, edges, poles and the coefficient table are required");
    NBK_CHECK_ARG(nedges >= 2 && nedges <= TP_MAX_NB + 1, "threeptcf: %d edges (2 .. %d supported: at most %d radial bins)",
                  nedges, TP_MAX_NB + 1, TP_MAX_NB);
    for (int k = 0; k < nedges; k++) {
        NBK_CHECK_ARG(isfinite(edges_host[k]) && edges_host[k] >= 0, "threeptcf: edges must be finite and non-negative");
        NBK_CHECK_ARG(k == 0 || edges_host[k] > edges_host[k - 1], "threeptcf: edges must increase strictly");
    }
    NBK_CHECK_ARG(npoles >= 1 && npoles <= TP_MAX_POLES, "threeptcf: %d poles (1 .. %d supported)", npoles, TP_MAX_POLES);
    TpParam t;
    t.L = 0;
    for (int i = 0; i < npoles; i++) {
        NBK_CHECK_ARG(poles_host[i] >= 0 && poles_host[i] <= TP_MAX_L, "threeptcf: pole %d out of range (0 .. %d supported)",
                      poles_host[i], TP_MAX_L);
        for (int j = 0; j < i; j++) NBK_CHECK_ARG(poles_host[j] != poles_host[i], "threeptcf: pole %d given twice", poles_host[i]);
        t.poles[i] = poles_host[i];
        if (poles_host[i] > t.L) t.L = poles_host[i];
    }
    t.nmom = (t.L + 1) * (t.L + 2) / 2;
    t.npole = npoles;
    t.nb = nedges - 1;
    t.nbp = t.nb * (t.nb + 1) / 2;
    for (int i = 0; i < t.nmom * (t.L + 1); i++)
        NBK_CHECK_ARG(isfinite(coef_host[i]), "threeptcf: the coefficient table must be finite");
    PcGeom g;
    g.mode = NBK_PC_1D;
    g.periodic = periodic ? 1 : 0;
    g.nb = t.nb;
    g.n2 = 1;
    g.pimax = 0.0;
    const double smax = edges_host[nedges - 1];
    // the skip thresholds: a relative margin far above the rounding of the gaps and of the separations
    g.thr_xy = smax * smax * (1.0 + 1e-9);
    g.thr_sph = g.thr_xy;
    double cells = 1.0;
    for (int d = 0; d < 3; d++) {
        NBK_CHECK_ARG(isfinite(box_host[d]) && box_host[d] > 0, "threeptcf: box side %d must be positive and finite", d);
        NBK_CHECK_ARG(ncell_host[d] >= 1 && ncell_host[d] <= TP_MAX_CELLS_PER_AXIS, "threeptcf: cell count %lld on axis %d out of range",
                      (long long)ncell_host[d], d);
        NBK_CHECK_ARG(isfinite(tol_host[d]) && tol_host[d] >= 0, "threeptcf: bad tolerance on axis %d", d);
        g.box[d] = box_host[d];
        g.nc[d] = ncell_host[d];
        g.cs[d] = box_host[d] / (double)ncell_host[d];
        g.tol[d] = tol_host[d];
        g.reach[d] = (long long)floor((smax + 2.0 * g.tol[d]) / g.cs[d] * (1.0 + 1e-12)) + 1;
        cells *= (double)ncell_host[d];
    }
    NBK_CHECK_ARG(cells < 9.2e18, "threeptcf: %g cells do not fit a 63-bit key", cells);
    const int ncoef = t.nmom * (t.L + 1);
    if (nchunks == 0 || nscells == 0) return NBK_OK;
    NBK_CHECK_ARG(work != nullptr && zeta != nullptr && npairs != nullptr && candidates != nullptr,
                  "threeptcf: a device workspace of %d doubles and the outputs are required", nedges + ncoef);
    int dev = 0, optin = 0;
    NBK_CUDA(cudaGetDevice(&dev));
    NBK_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    // as many warps (primaries per round) as shared memory holds
    t.nw = 0;
    for (int nw = TP_MAX_NW; nw >= 1; nw--)
        if (tp_smem(nw, t.nb, t.nmom, t.L, npoles) <= (size_t)optin) { t.nw = nw; break; }
    NBK_CHECK_ARG(t.nw >= 1, "threeptcf: %zu bytes of shared memory needed, %d available", tp_smem(1, t.nb, t.nmom, t.L, npoles), optin);
    const size_t shm = tp_smem(t.nw, t.nb, t.nmom, t.L, npoles);
    cudaStream_t s = (cudaStream_t)stream;
    double *hbuf = (double *)malloc(sizeof(double) * (nedges + ncoef));
    NBK_CHECK_ARG(hbuf != nullptr, "threeptcf: out of host memory");
    for (int k = 0; k < nedges; k++) hbuf[k] = edges_host[k];
    for (int k = 0; k < ncoef; k++) hbuf[nedges + k] = coef_host[k];
    cudaError_t e = cudaMemcpyAsync(work, hbuf, sizeof(double) * (nedges + ncoef), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    free(hbuf);
    NBK_CUDA(e);
    if (shm > 48 * 1024) NBK_CUDA(cudaFuncSetAttribute(k_threeptcf, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
    k_threeptcf<<<(unsigned)nchunks, 32 * t.nw, shm, s>>>(
        ppos, pw, (const long long *)chunk_first, (const long long *)chunk_key, spos, sw, (const unsigned *)scell_start,
        (const long long *)scell_key, nscells, g, t, work, work + nedges, zeta, (unsigned long long *)npairs,
        (unsigned long long *)candidates);
    NBK_LAUNCHED();
    return NBK_OK;
}
