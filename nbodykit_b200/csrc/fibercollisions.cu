// Fiber collisions (nbodykit/algorithms/fibercollisions.py: FiberCollisions; DESIGN.md 4.11) on the members of the
// angular FOF groups, sorted by (label, global row) into group segments.
//   nbk_fc_pairs     : groups of 2: the hashed pick of the two is collided, its neighbour is the other
//   nbk_fc_small     : groups of 3 .. 32, one warp each: collision masks, the greedy and the nearest uncollided member
//                      in registers
//   nbk_fc_cell_keys : the cell of every member of a larger group, on a grid of cells of side >= rad
//   nbk_fc_count / nbk_fc_write : per member of a larger group, its colliding members (group-local indices) from the
//                      3 x 3 x 3 cells around it, as CSR lists (count, then write)
//   nbk_fc_greedy    : larger groups, one block each: the greedy with incremental counts, in shared memory up to
//                      nbk_fc_smem_members() members, in global scratch beyond
//   nbk_fc_nearest   : per collided member of a larger group, the nearest uncollided member by a walk over rings of cells
// Members a, b collide when d <= rad, d = sqrt((dx^2 + dy^2) + dz^2) in double from the float32 positions.  The greedy
// removes, among the alive members with the most alive colliders (n_coll), those whose colliders have the fewest
// colliders in all (n_other), the hashed pick; it stops when no alive member has a collider.  The file is compiled with
// --fmad=false: no contraction may move a pair across the collision radius.
#include "pc_cells.cuh"

#include <climits>
#include <math.h>

#define FC_WARP_MAX 32
#define FC_GB 256
#define FC_LB 128
#define FC_SMEM_MEMBERS 2048

// SplitMix64 finaliser; the pick of removal `step` of the group whose smallest global row is g, among k candidates in
// member order, is ((h >> 32) * k) >> 32 with h = mix(mix(mix(seed) ^ g) ^ step)
static __host__ __device__ __forceinline__ unsigned long long fc_mix(unsigned long long z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

static __device__ __forceinline__ unsigned fc_pick(unsigned long long seed, long long g, long long step, unsigned k) {
    const unsigned long long h = fc_mix(fc_mix(fc_mix(seed) ^ (unsigned long long)g) ^ (unsigned long long)step);
    return (unsigned)(((h >> 32) * (unsigned long long)k) >> 32);
}

static __device__ __forceinline__ double fc_dist(float ax, float ay, float az, float bx, float by, float bz) {
    const double dx = (double)ax - (double)bx, dy = (double)ay - (double)by, dz = (double)az - (double)bz;
    return sqrt((dx * dx + dy * dy) + dz * dz);
}

__global__ void k_fc_pairs(const long long *__restrict__ gstart, const int *__restrict__ gid, long long ng,
                           const long long *__restrict__ grow, unsigned long long seed, int *__restrict__ collided,
                           long long *__restrict__ neighbor) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < ng; t += stride) {
        const long long s = gstart[gid[t]];
        const unsigned c = fc_pick(seed, grow[s], 0, 2u);
        collided[s + c] = 1;
        neighbor[s + c] = grow[s + (c ^ 1u)];
    }
}

// one warp per group of 3 .. 32 members; lane m holds member m
__global__ void k_fc_small(const float *__restrict__ pos, const long long *__restrict__ gstart, const int *__restrict__ gid,
                           long long ng, const long long *__restrict__ grow, double rad, unsigned long long seed,
                           int *__restrict__ collided, long long *__restrict__ neighbor, unsigned long long *__restrict__ steps) {
    const int lane = threadIdx.x & 31;
    const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= ng) return;
    const long long s = gstart[gid[w]];
    const int N = (int)(gstart[gid[w] + 1] - s);
    const bool in = lane < N;
    float px = 0.f, py = 0.f, pz = 0.f;
    long long row = 0;
    if (in) { px = pos[3 * (s + lane)]; py = pos[3 * (s + lane) + 1]; pz = pos[3 * (s + lane) + 2]; row = grow[s + lane]; }
    unsigned mask = 0;
    for (int j = 0; j < N; j++) {
        const float qx = __shfl_sync(0xffffffffu, px, j), qy = __shfl_sync(0xffffffffu, py, j), qz = __shfl_sync(0xffffffffu, pz, j);
        if (in && j != lane && fc_dist(px, py, pz, qx, qy, qz) <= rad) mask |= 1u << j;
    }
    const long long g = __shfl_sync(0xffffffffu, row, 0);
    unsigned alive = N == 32 ? 0xffffffffu : ((1u << N) - 1u);
    bool coll = false;
    long long step = 0;
    while (true) {
        const bool a = in && ((alive >> lane) & 1u);
        const unsigned am = mask & alive;
        const int nc = a ? __popc(am) : -1;
        long long no = 0;
        for (int j = 0; j < N; j++) {
            const int v = __shfl_sync(0xffffffffu, nc, j);
            if ((am >> j) & 1u) no += v;
        }
        // the most colliders, then the fewest colliders of colliders
        int bnc = nc;
        long long bno = a ? no : LLONG_MAX;
        for (int o = 16; o > 0; o >>= 1) {
            const int onc = __shfl_xor_sync(0xffffffffu, bnc, o);
            const long long ono = __shfl_xor_sync(0xffffffffu, bno, o);
            if (onc > bnc || (onc == bnc && ono < bno)) { bnc = onc; bno = ono; }
        }
        if (bnc <= 0) break;
        unsigned cand = __ballot_sync(0xffffffffu, a && nc == bnc && no == bno);
        const unsigned pick = fc_pick(seed, g, step, (unsigned)__popc(cand));
        for (unsigned k = 0; k < pick; k++) cand &= cand - 1u;
        const int c = __ffs(cand) - 1;
        alive &= ~(1u << c);
        if (lane == c) coll = true;
        step++;
    }
    if (lane == 0 && step) atomicAdd(steps, (unsigned long long)step);
    // the nearest uncollided member; the first in member order on a tie
    const unsigned unc = __ballot_sync(0xffffffffu, in && !coll);
    double bd = INFINITY;
    long long bn = -1;
    for (int j = 0; j < N; j++) {
        const float qx = __shfl_sync(0xffffffffu, px, j), qy = __shfl_sync(0xffffffffu, py, j), qz = __shfl_sync(0xffffffffu, pz, j);
        const long long r = __shfl_sync(0xffffffffu, row, j);
        if (!((unc >> j) & 1u)) continue;
        const double d = fc_dist(px, py, pz, qx, qy, qz);
        if (d < bd) { bd = d; bn = r; }
    }
    if (in && coll) {
        collided[s + lane] = 1;
        neighbor[s + lane] = bn;
    }
}

struct FcGrid {
    double cs;
    long long nc;
};

static __device__ __forceinline__ long long fc_cell(float x, const FcGrid &g) {
    long long c = (long long)floor((double)x / g.cs);
    return c < 0 ? 0 : (c >= g.nc ? g.nc - 1 : c);
}

__global__ void k_fc_cell_keys(const float *__restrict__ pos, const long long *__restrict__ lrow, long long nl, FcGrid g,
                               long long *__restrict__ keys) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nl; i += stride) {
        const long long s = lrow[i];
        keys[i] = (fc_cell(pos[3 * s], g) * g.nc + fc_cell(pos[3 * s + 1], g)) * g.nc + fc_cell(pos[3 * s + 2], g);
    }
}

// The members of larger groups are numbered l = lbeg[q] + m (member m of larger group q, whose segment starts at
// lseg[q]); cidx / ckey are those l sorted by (q, cell key).  WRITE = false: cnt[l] = colliders of l; WRITE = true: their
// group-local indices at nbr[off[l] ..].
template <bool WRITE>
__global__ void __launch_bounds__(FC_LB) k_fc_lists(const float *__restrict__ pos, const int *__restrict__ lq,
                                                   const long long *__restrict__ lbeg, const long long *__restrict__ lseg, long long nl,
                                                   const int *__restrict__ cidx, const long long *__restrict__ ckey, FcGrid g,
                                                   double rad, long long *__restrict__ cnt, const long long *__restrict__ off,
                                                   int *__restrict__ nbr, unsigned long long *__restrict__ g_cand) {
    const long long l = (long long)blockIdx.x * FC_LB + threadIdx.x;
    unsigned long long cand = 0;
    if (l < nl) {
        const int q = lq[l];
        const long long b = lbeg[q], N = lbeg[q + 1] - b, s = lseg[q], m = l - b;
        const float px = pos[3 * (s + m)], py = pos[3 * (s + m) + 1], pz = pos[3 * (s + m) + 2];
        const long long ix = fc_cell(px, g), iy = fc_cell(py, g), iz = fc_cell(pz, g);
        const long long z0 = iz > 0 ? iz - 1 : 0, z1 = iz + 1 < g.nc ? iz + 1 : g.nc - 1;
        long long found = 0, w = WRITE ? off[l] : 0;
        for (long long x = ix - 1; x <= ix + 1; x++) {
            if (x < 0 || x >= g.nc) continue;
            for (long long y = iy - 1; y <= iy + 1; y++) {
                if (y < 0 || y >= g.nc) continue;
                const long long row = (x * g.nc + y) * g.nc;
                const long long e0 = pc_lower_bound(ckey + b, N, row + z0), e1 = pc_lower_bound(ckey + b, N, row + z1 + 1);
                cand += (unsigned long long)(e1 - e0);
                for (long long e = e0; e < e1; e++) {
                    const long long mj = cidx[b + e] - b;
                    if (mj == m) continue;
                    const long long sj = s + mj;
                    if (!(fc_dist(px, py, pz, pos[3 * sj], pos[3 * sj + 1], pos[3 * sj + 2]) <= rad)) continue;
                    if (WRITE) nbr[w + found] = (int)mj;
                    found++;
                }
            }
        }
        if (!WRITE) cnt[l] = found;
    }
    if (!WRITE) {
        for (int o = 16; o > 0; o >>= 1) cand += __shfl_down_sync(0xffffffffu, cand, o);
        if ((threadIdx.x & 31) == 0 && cand) atomicAdd(g_cand, cand);
    }
}

struct FcBest {
    int nc;
    long long no;
};

static __device__ __forceinline__ FcBest fc_better(FcBest a, FcBest b) {
    return (b.nc > a.nc || (b.nc == a.nc && b.no < a.no)) ? b : a;
}

// the block-wide best (nc, no): every thread gets it
static __device__ FcBest fc_block_best(FcBest v, FcBest *red) {
    for (int o = 16; o > 0; o >>= 1) {
        FcBest u;
        u.nc = __shfl_xor_sync(0xffffffffu, v.nc, o);
        u.no = __shfl_xor_sync(0xffffffffu, v.no, o);
        v = fc_better(v, u);
    }
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) red[wid] = v;
    __syncthreads();
    FcBest r = red[0];
    for (int k = 1; k < FC_GB / 32; k++) r = fc_better(r, red[k]);
    return r;
}

// exclusive prefix of v over the threads of the block, and the total
static __device__ long long fc_block_scan(long long v, long long *red, long long &total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    long long x = v;
    for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    __syncthreads();
    if (lane == 31) red[wid] = x;
    __syncthreads();
    long long before = 0;
    total = 0;
    for (int k = 0; k < FC_GB / 32; k++) {
        if (k < wid) before += red[k];
        total += red[k];
    }
    return before + x - v;
}

// One block per larger group.  n_coll[i] = alive colliders of i, n_other[i] = the sum of n_coll over them.  Removing c
// (n_coll M): every alive collider j of c loses 1 from n_coll and M from n_other, and every alive collider k of such a j
// loses 1 from n_other -- exact integer updates, so the state equals a recount at every step.
__global__ void __launch_bounds__(FC_GB) k_fc_greedy(const long long *__restrict__ lbeg, const long long *__restrict__ lseg,
                                                    long long nlg, const long long *__restrict__ off, const int *__restrict__ nbr,
                                                    const long long *__restrict__ grow, unsigned long long seed,
                                                    int *__restrict__ g_ncoll, long long *__restrict__ g_nother,
                                                    unsigned char *__restrict__ g_alive, int *__restrict__ collided,
                                                    long long *__restrict__ nunc, unsigned long long *__restrict__ steps) {
    extern __shared__ long long fc_smem[];
    __shared__ FcBest red_best[FC_GB / 32];
    __shared__ long long red_scan[FC_GB / 32];
    __shared__ int chosen;
    const long long q = blockIdx.x;
    const long long b = lbeg[q], N = lbeg[q + 1] - b, s = lseg[q];
    const long long *o = off + b;
    long long *nother;
    int *ncoll;
    unsigned char *alive;
    if (N <= FC_SMEM_MEMBERS) {
        nother = fc_smem;
        ncoll = (int *)(fc_smem + N);
        alive = (unsigned char *)(ncoll + N);
    } else {
        nother = g_nother + b;
        ncoll = g_ncoll + b;
        alive = g_alive + b;
    }
    for (long long m = threadIdx.x; m < N; m += FC_GB) {
        ncoll[m] = (int)(o[m + 1] - o[m]);
        alive[m] = 1;
    }
    __syncthreads();
    for (long long m = threadIdx.x; m < N; m += FC_GB) {
        long long t = 0;
        for (long long e = o[m]; e < o[m + 1]; e++) t += ncoll[nbr[e]];
        nother[m] = t;
    }
    __syncthreads();
    const long long g = grow[s];
    const long long chunk = (N + FC_GB - 1) / FC_GB;
    const long long m0 = threadIdx.x * chunk, m1 = m0 + chunk < N ? m0 + chunk : N;
    long long step = 0, ncol = 0;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    while (true) {
        FcBest v{-1, LLONG_MAX};
        for (long long m = m0; m < m1; m++)
            if (alive[m]) v = fc_better(v, FcBest{ncoll[m], nother[m]});
        const FcBest best = fc_block_best(v, red_best);
        if (best.nc <= 0) break;
        long long k = 0;
        for (long long m = m0; m < m1; m++) k += (alive[m] && ncoll[m] == best.nc && nother[m] == best.no) ? 1 : 0;
        long long total;
        const long long before = fc_block_scan(k, red_scan, total);
        const long long pick = (long long)fc_pick(seed, g, step, (unsigned)total);
        if (pick >= before && pick < before + k) {
            long long r = pick - before;
            for (long long m = m0; m < m1; m++) {
                if (alive[m] && ncoll[m] == best.nc && nother[m] == best.no) {
                    if (r == 0) { chosen = (int)m; break; }
                    r--;
                }
            }
        }
        __syncthreads();
        const int c = chosen;
        if (threadIdx.x == 0) {
            alive[c] = 0;
            collided[s + c] = 1;
        }
        __syncthreads();
        // one warp per collider j of c, its lanes over the colliders of j
        for (long long e = o[c] + wid; e < o[c + 1]; e += FC_GB / 32) {
            const int j = nbr[e];
            if (!alive[j]) continue;
            if (lane == 0) {
                ncoll[j] -= 1;
                atomicAdd((unsigned long long *)&nother[j], (unsigned long long)(-(long long)best.nc));
            }
            for (long long f = o[j] + lane; f < o[j + 1]; f += 32) {
                const int kk = nbr[f];
                if (alive[kk]) atomicAdd((unsigned long long *)&nother[kk], (unsigned long long)(-1ll));
            }
        }
        __syncthreads();
        step++;
        ncol++;
    }
    if (threadIdx.x == 0) {
        nunc[q] = N - ncol;
        if (step) atomicAdd(steps, (unsigned long long)step);
    }
}

// one thread per member of a larger group; collided members walk Chebyshev rings of cells around their own until every
// uncollided member has been seen or the next ring cannot hold a nearer one
__global__ void __launch_bounds__(FC_LB) k_fc_nearest(const float *__restrict__ pos, const int *__restrict__ lq,
                                                     const long long *__restrict__ lbeg, const long long *__restrict__ lseg,
                                                     long long nl, const int *__restrict__ cidx, const long long *__restrict__ ckey,
                                                     FcGrid g, const int *__restrict__ collided, const long long *__restrict__ nunc,
                                                     const long long *__restrict__ grow, long long *__restrict__ neighbor) {
    const long long l = (long long)blockIdx.x * FC_LB + threadIdx.x;
    if (l >= nl) return;
    const int q = lq[l];
    const long long b = lbeg[q], N = lbeg[q + 1] - b, s = lseg[q], m = l - b;
    if (!collided[s + m]) return;
    const float px = pos[3 * (s + m)], py = pos[3 * (s + m) + 1], pz = pos[3 * (s + m) + 2];
    const long long ix = fc_cell(px, g), iy = fc_cell(py, g), iz = fc_cell(pz, g);
    const long long nu = nunc[q];
    double bd = INFINITY;
    long long bm = LLONG_MAX, seen = 0;
    for (long long R = 0; R <= g.nc; R++) {
        for (long long x = ix - R; x <= ix + R; x++) {
            if (x < 0 || x >= g.nc) continue;
            for (long long y = iy - R; y <= iy + R; y++) {
                if (y < 0 || y >= g.nc) continue;
                const bool face = x == ix - R || x == ix + R || y == iy - R || y == iy + R;
                const long long row = (x * g.nc + y) * g.nc;
                for (int part = 0; part < (face ? 1 : 2); part++) {
                    long long za, zb;
                    if (face) { za = iz - R; zb = iz + R; }
                    else { za = zb = part ? iz + R : iz - R; }
                    za = za < 0 ? 0 : za;
                    zb = zb >= g.nc ? g.nc - 1 : zb;
                    if (za > zb) continue;
                    const long long e0 = pc_lower_bound(ckey + b, N, row + za), e1 = pc_lower_bound(ckey + b, N, row + zb + 1);
                    for (long long e = e0; e < e1; e++) {
                        const long long mj = cidx[b + e] - b;
                        const long long sj = s + mj;
                        if (collided[sj]) continue;
                        seen++;
                        const double d = fc_dist(px, py, pz, pos[3 * sj], pos[3 * sj + 1], pos[3 * sj + 2]);
                        if (d < bd || (d == bd && mj < bm)) { bd = d; bm = mj; }
                    }
                }
            }
        }
        if (seen >= nu) break;
        // every cell of ring R + 1 lies at least R cell sides away
        if ((double)R * g.cs * (1.0 - 1e-9) > bd) break;
    }
    neighbor[s + m] = grow[s + bm];
}

static int fc_grid(FcGrid &g, double cs, int64_t nc) {
    NBK_CHECK_ARG(isfinite(cs) && cs > 0, "fibercollisions: the cell side must be positive and finite (got %g)", cs);
    NBK_CHECK_ARG(nc >= 1 && nc <= (1ll << 21), "fibercollisions: %lld cells per axis out of range", (long long)nc);
    g.cs = cs;
    g.nc = nc;
    return NBK_OK;
}

extern "C" int64_t nbk_fc_warp_members(void) { return FC_WARP_MAX; }
extern "C" int64_t nbk_fc_smem_members(void) { return FC_SMEM_MEMBERS; }

extern "C" int nbk_fc_pairs(const int64_t *gstart, const int32_t *gid, int64_t ng, const int64_t *grow, uint64_t seed,
                            int32_t *collided, int64_t *neighbor, void *stream) {
    NBK_CHECK_ARG(ng >= 0 && ng < (1ll << 31), "fibercollisions: %lld groups out of range", (long long)ng);
    if (ng == 0) return NBK_OK;
    NBK_CHECK_ARG(gstart && gid && grow && collided && neighbor, "fibercollisions: null device array");
    cudaStream_t st = (cudaStream_t)stream;
    k_fc_pairs<<<nbk_grid_for(ng, 256, 8), 256, 0, st>>>((const long long *)gstart, gid, ng, (const long long *)grow, seed,
                                                         collided, (long long *)neighbor);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_fc_small(const float *pos, const int64_t *gstart, const int32_t *gid, int64_t ng, const int64_t *grow,
                            double rad, uint64_t seed, int32_t *collided, int64_t *neighbor, uint64_t *steps, void *stream) {
    NBK_CHECK_ARG(ng >= 0 && ng < (1ll << 31), "fibercollisions: %lld groups out of range", (long long)ng);
    NBK_CHECK_ARG(isfinite(rad) && rad > 0, "fibercollisions: the radius must be positive and finite (got %g)", rad);
    if (ng == 0) return NBK_OK;
    NBK_CHECK_ARG(pos && gstart && gid && grow && collided && neighbor && steps, "fibercollisions: null device array");
    cudaStream_t st = (cudaStream_t)stream;
    const long long blocks = (ng * 32 + 255) / 256;
    k_fc_small<<<(unsigned)blocks, 256, 0, st>>>(pos, (const long long *)gstart, gid, ng, (const long long *)grow, rad, seed,
                                                 collided, (long long *)neighbor, (unsigned long long *)steps);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_fc_cell_keys(const float *pos, const int64_t *lrow, int64_t nl, double cs, int64_t nc, int64_t *keys,
                                void *stream) {
    FcGrid g;
    int rc = fc_grid(g, cs, nc);
    if (rc) return rc;
    NBK_CHECK_ARG(nl >= 0 && nl < (1ll << 31), "fibercollisions: %lld members out of range", (long long)nl);
    if (nl == 0) return NBK_OK;
    NBK_CHECK_ARG(pos && lrow && keys, "fibercollisions: null device array");
    cudaStream_t st = (cudaStream_t)stream;
    k_fc_cell_keys<<<nbk_grid_for(nl, 256, 8), 256, 0, st>>>(pos, (const long long *)lrow, nl, g, (long long *)keys);
    NBK_LAUNCHED();
    return NBK_OK;
}

static int fc_lists(bool write, const float *pos, const int32_t *lq, const int64_t *lbeg, const int64_t *lseg, int64_t nl,
                    const int32_t *cidx, const int64_t *ckey, double cs, int64_t nc, double rad, int64_t *counts,
                    const int64_t *offsets, int32_t *nbr, uint64_t *candidates, void *stream) {
    FcGrid g;
    int rc = fc_grid(g, cs, nc);
    if (rc) return rc;
    NBK_CHECK_ARG(isfinite(rad) && rad > 0 && rad <= cs, "fibercollisions: the radius must be positive, finite and at most the "
                  "cell side (got %g, cell side %g)", rad, cs);
    NBK_CHECK_ARG(nl >= 0 && nl < (1ll << 31), "fibercollisions: %lld members out of range", (long long)nl);
    if (nl == 0) return NBK_OK;
    NBK_CHECK_ARG(pos && lq && lbeg && lseg && cidx && ckey, "fibercollisions: null device array");
    NBK_CHECK_ARG(write ? (offsets && nbr) : (counts && candidates), "fibercollisions: null output array");
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned blocks = (unsigned)((nl + FC_LB - 1) / FC_LB);
    if (write)
        k_fc_lists<true><<<blocks, FC_LB, 0, st>>>(pos, lq, (const long long *)lbeg, (const long long *)lseg, nl, cidx,
                                                   (const long long *)ckey, g, rad, nullptr, (const long long *)offsets, nbr, nullptr);
    else
        k_fc_lists<false><<<blocks, FC_LB, 0, st>>>(pos, lq, (const long long *)lbeg, (const long long *)lseg, nl, cidx,
                                                    (const long long *)ckey, g, rad, (long long *)counts, nullptr, nullptr,
                                                    (unsigned long long *)candidates);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_fc_count(const float *pos, const int32_t *lq, const int64_t *lbeg, const int64_t *lseg, int64_t nl,
                            const int32_t *cidx, const int64_t *ckey, double cs, int64_t nc, double rad, int64_t *counts,
                            uint64_t *candidates, void *stream) {
    return fc_lists(false, pos, lq, lbeg, lseg, nl, cidx, ckey, cs, nc, rad, counts, nullptr, nullptr, candidates, stream);
}

extern "C" int nbk_fc_write(const float *pos, const int32_t *lq, const int64_t *lbeg, const int64_t *lseg, int64_t nl,
                            const int32_t *cidx, const int64_t *ckey, double cs, int64_t nc, double rad, const int64_t *offsets,
                            int32_t *nbr, void *stream) {
    return fc_lists(true, pos, lq, lbeg, lseg, nl, cidx, ckey, cs, nc, rad, nullptr, offsets, nbr, nullptr, stream);
}

extern "C" int nbk_fc_greedy(const int64_t *lbeg, const int64_t *lseg, int64_t nlg, int64_t max_members, const int64_t *offsets,
                             const int32_t *nbr, const int64_t *grow, uint64_t seed, int32_t *scratch_ncoll,
                             int64_t *scratch_nother, uint8_t *scratch_alive, int32_t *collided, int64_t *nunc, uint64_t *steps,
                             void *stream) {
    NBK_CHECK_ARG(nlg >= 0 && nlg < (1ll << 31), "fibercollisions: %lld groups out of range", (long long)nlg);
    NBK_CHECK_ARG(max_members >= 0 && max_members < (1ll << 31), "fibercollisions: group size %lld out of range",
                  (long long)max_members);
    if (nlg == 0) return NBK_OK;
    NBK_CHECK_ARG(lbeg && lseg && offsets && nbr && grow && collided && nunc && steps, "fibercollisions: null device array");
    NBK_CHECK_ARG(max_members <= FC_SMEM_MEMBERS || (scratch_ncoll && scratch_nother && scratch_alive),
                  "fibercollisions: groups above %d members need the global scratch", FC_SMEM_MEMBERS);
    const long long ms = max_members < FC_SMEM_MEMBERS ? max_members : FC_SMEM_MEMBERS;
    const size_t smem = (size_t)ms * 13 + 8;
    cudaStream_t st = (cudaStream_t)stream;
    k_fc_greedy<<<(unsigned)nlg, FC_GB, smem, st>>>((const long long *)lbeg, (const long long *)lseg, nlg,
                                                   (const long long *)offsets, nbr, (const long long *)grow, seed, scratch_ncoll,
                                                   (long long *)scratch_nother, scratch_alive, collided, (long long *)nunc,
                                                   (unsigned long long *)steps);
    NBK_LAUNCHED();
    return NBK_OK;
}

extern "C" int nbk_fc_nearest(const float *pos, const int32_t *lq, const int64_t *lbeg, const int64_t *lseg, int64_t nl,
                              const int32_t *cidx, const int64_t *ckey, double cs, int64_t nc, const int32_t *collided,
                              const int64_t *nunc, const int64_t *grow, int64_t *neighbor, void *stream) {
    FcGrid g;
    int rc = fc_grid(g, cs, nc);
    if (rc) return rc;
    NBK_CHECK_ARG(nl >= 0 && nl < (1ll << 31), "fibercollisions: %lld members out of range", (long long)nl);
    if (nl == 0) return NBK_OK;
    NBK_CHECK_ARG(pos && lq && lbeg && lseg && cidx && ckey && collided && nunc && grow && neighbor,
                  "fibercollisions: null device array");
    cudaStream_t st = (cudaStream_t)stream;
    k_fc_nearest<<<(unsigned)((nl + FC_LB - 1) / FC_LB), FC_LB, 0, st>>>(pos, lq, (const long long *)lbeg, (const long long *)lseg,
                                                                        nl, cidx, (const long long *)ckey, g, collided,
                                                                        (const long long *)nunc, (const long long *)grow,
                                                                        (long long *)neighbor);
    NBK_LAUNCHED();
    return NBK_OK;
}
