/*
 * nbk_b200 -- C ABI of the H100-native FFTPower hot path (libnbk_b200.so).
 *
 * The reference (bccp/nbodykit) has no C ABI of its own: its seam for this path is the
 * duck-typed Python interface of the un-vendored `pmesh` package.  Each entry point
 * below names the reference call site(s) whose arithmetic it replaces (paths relative to
 * the nbodykit tree).  All pointers are DEVICE pointers unless marked `host`; sizes are
 * element counts; every call is asynchronous and ordered on `stream` (a cudaStream_t
 * passed as void*, NULL = legacy default stream).  Return value: 0 on success, negative
 * on error (nbk_last_error() gives the text).  No torch types, no C++ exceptions cross
 * this boundary.
 */
#ifndef NBK_B200_H
#define NBK_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* scalar type codes */
#define NBK_F4 4
#define NBK_F8 8

/* resampling windows: value == support (pmesh.window.methods[...].support,
 * source/mesh/catalog.py:194,271-273) */
#define NBK_WINDOW_NNB 1
#define NBK_WINDOW_CIC 2
#define NBK_WINDOW_TSC 3
#define NBK_WINDOW_PCS 4

/* compensation transfer functions (source/mesh/catalog.py:449-594) */
/* layout bits of the `transposed` argument of the Fourier-space entry points */
#define NBK_LAYOUT_TRANSPOSED 1  /* first stored axis is y: [y_n][Nx][Nzc] (what one slab transpose leaves behind) */
#define NBK_LAYOUT_FULLZ 2       /* the last axis stores all Nz modes (complex-dtype meshes, ComplexField.compressed
                                    == False, algorithms/fftpower.py:572) instead of the Hermitian half Nz/2+1 */

#define NBK_COMP_NONE 0
#define NBK_COMP_CIC 1           /* CompensateCIC            :513-535 */
#define NBK_COMP_TSC 2           /* CompensateTSC            :449-473 */
#define NBK_COMP_PCS 3           /* CompensatePCS            :475-500 */
#define NBK_COMP_CIC_SHOTNOISE 4 /* CompensateCICShotnoise   :573-594 */
#define NBK_COMP_TSC_SHOTNOISE 5 /* CompensateTSCShotnoise   :537-559 */
#define NBK_COMP_PCS_SHOTNOISE 6 /* CompensatePCSShotnoise   :561-571 */

/* error codes */
#define NBK_OK 0
#define NBK_ERR_ARG -1
#define NBK_ERR_CUDA -2
#define NBK_ERR_UNSUPPORTED -3

int nbk_version(void);
const char *nbk_last_error(void);
/* number of kernels this library has launched since load (bench.py's "gpu_launches") */
int64_t nbk_launch_count(void);

/* ---------------------------------------------------------------------------------------
 * Layout of a (slab of a) mesh.  Real field: x-major C order [x_n][Ny][Nz].  Complex field:
 * Hermitian-compressed on the last axis, Nzc = Nz/2+1.  `transposed == 0`: [x_n][Ny][Nzc]
 * holding x planes [x_start, x_start+x_n);  `transposed == 1`: [y_n][Nx][Nzc] holding y rows
 * [y_start, y_start+y_n) of every x (what the slab FFT leaves on each GPU when P > 1).
 * ------------------------------------------------------------------------------------- */

/* pm.paint(pos, mass=, resampler=, transform=pm.affine[.shift(s)], hold=True, out=)
 * -- source/mesh/catalog.py:287,295-296 (pmesh window scatter).
 * pos: [n][3] row-major, pos_dtype F4|F8.  mass: [n] or NULL (unit), mass_dtype F4|F8.
 * Grid coordinate g_d = fl(fl(double(pos_d)*fl(N_d/L_d)) + shift) (no FMA), periodic wrap in
 * grid units; stencil points whose x plane is outside [x_start, x_start+x_n) are dropped
 * (pmesh ghost semantics).  Always accumulates into `mesh` (hold=True); zero it first
 * with nbk_fill for hold=False.  mesh_dtype F4|F8. */
int nbk_paint(const void *pos, int pos_dtype, int64_t n, const void *mass, int mass_dtype,
              int window, double shift, const double *boxsize_host, const int64_t *nmesh_host,
              int64_t x_start, int64_t x_n, void *mesh, int mesh_dtype, void *stream);

/* same, painting the un-shifted and the +0.5-cell shifted mesh in one pass over the particles
 * (the interlaced branch, source/mesh/catalog.py:289-296) */
int nbk_paint_interlaced(const void *pos, int pos_dtype, int64_t n, const void *mass,
                         int mass_dtype, int window, const double *boxsize_host,
                         const int64_t *nmesh_host, int64_t x_start, int64_t x_n, void *mesh1,
                         void *mesh2, int mesh_dtype, void *stream);

/* The same scatter through the tile-sorted path: particles are bucketed by 16^3-cell tile, each tile is
 * accumulated in shared memory in 64-bit fixed point (order-independent, resolution 2^-31 of the largest
 * |mass|) and flushed once.  mesh2 != NULL paints the +0.5-cell shifted mesh of the interlaced branch from
 * the same buckets (then shift must be 0).  `work`: device scratch of nbk_paint_tiled_workspace() bytes.
 * clear != 0 gives pm.paint(hold=False): the mesh(es) are zeroed by the call itself (inside the bucketing
 * pass, no separate fill); clear == 0 accumulates into what is there (hold=True).
 * nbk_paint_tiled_supported() says whether the mesh admits the tiling (sides multiples of 16, >= 32). */
int nbk_paint_tiled_supported(const int64_t *nmesh_host, int64_t x_n, int window);
int64_t nbk_paint_tiled_workspace(int64_t n, int pos_dtype, int mass_dtype, const int64_t *nmesh_host,
                                  int64_t x_n);
int nbk_paint_tiled(const void *pos, int pos_dtype, int64_t n, const void *mass, int mass_dtype, int window,
                    double shift, const double *boxsize_host, const int64_t *nmesh_host, int64_t x_start,
                    int64_t x_n, void *mesh, void *mesh2, int mesh_dtype, void *work, int64_t work_bytes,
                    int clear, void *stream);

/* pm.decompose(pos, smoothing) + Layout.exchange (source/mesh/catalog.py:271-284) for the x-slab decomposition:
 * nbk_route_count finds the particles with a plane within `smoothing` cells (periodic) owned by ANOTHER rank
 * (P <= 32) and appends one entry per such particle to `list` (device uint64[n] capacity, any order):
 * index in the low 32 bits, destination bitmask in the high 32 bits.  `counts`: device uint64[P+1], zero first;
 * [0..P) receive the per-destination counts, [P] the number of list entries.
 * nbk_route_scatter copies (pos[, mass]) of the listed particles into per-destination segments of a send
 * buffer (`offsets`: device int64[P] exclusive scan of the counts; `cursor`: device uint64[P], zero first);
 * `send_index` (optional, device int64[sum counts]) receives the source row of every sent row, so that per-row
 * results computed by the destination (readout partial sums) can be added back after the return all-to-all.
 * Local particles are never copied: each rank paints its own array plus what it receives. */
int nbk_route_count(const void *pos, int pos_dtype, int64_t n, double smoothing, const double *boxsize_host,
                    const int64_t *nmesh_host, int P, int rank, uint64_t *counts, uint64_t *list, void *stream);
int nbk_route_scatter(const void *pos, int pos_dtype, const void *mass, int mass_dtype, const uint64_t *list,
                      int64_t n_list, int P, const int64_t *offsets, uint64_t *cursor, void *send_pos,
                      void *send_mass, int64_t *send_index, void *stream);

/* RealField.readout(pos, resampler=, transform=, out=) (pmesh; called from algorithms/fftrecon.py:239-244): the gather
 * transposed to nbk_paint -- out[p] (= or +=, `accumulate`) sum over the stencil of W * mesh[cell], same grid
 * coordinate / window / slab semantics (planes outside [x_start, x_start+x_n) contribute nothing: per-rank partial
 * sums).  out: device [n] of out_dtype. */
int nbk_readout(const void *mesh, int mesh_dtype, const void *pos, int pos_dtype, int64_t n, int window, double shift,
                const double *boxsize_host, const int64_t *nmesh_host, int64_t x_start, int64_t x_n, void *out,
                int out_dtype, int accumulate, void *stream);

/* reconstruction displacement modes (algorithms/fftrecon.py:213-230, Field.apply(kernel(d), kind='wavenumber')):
 * out = i k_axis / k^2 * in * exp(-k^2 R^2 / 2) / (bias (1 + f/bias mu^2)), mu = k.los/|k|, the k = 0 mode -> 0.
 * Out of place on the Hermitian-compressed field (same layout flags as nbk_compensate). */
int nbk_recon_displacement(const void *in, void *out, int dtype, const int64_t *nmesh_host, const double *boxsize_host,
                           int transposed, int64_t start, int64_t count, int axis, double R, double bias, double f,
                           const double *los_host, void *stream);

/* leftmost stencil cell (wrapped) of every particle, [n][3] int32 -- the bit-exact part of the
 * paint contract, exported for parity tests and for pm.decompose (catalog.py:271-273) */
int nbk_cell_index(const void *pos, int pos_dtype, int64_t n, int window, double shift,
                   const double *boxsize_host, const int64_t *nmesh_host, int32_t *cell_out,
                   void *stream);

/* Wlocal = sum w, W2local = sum w^2 (source/mesh/catalog.py:265-267); out2: device double[2],
 * accumulated into (zero it first). */
int nbk_sum_w_w2(const void *w, int dtype, int64_t n, double *out2, void *stream);

/* RealField.r2c / ComplexField.c2r (base/mesh.py:228,237; source/mesh/catalog.py:341-351).
 * Forward is normalised by 1/(Nx*Ny*Nz), backward unnormalised (source/mesh/array.py:36-37).
 * Single-GPU whole-mesh transforms; real [Nx][Ny][Nz], cplx [Nx][Ny][Nzc].  Out of place.
 * Limits: every side a power of two, Nz >= 4; Nx, Ny <= 8192 and Nz <= 16384 in f4, Nx, Ny <= 4096 and Nz <= 8192 in
 * f8 (one CTA holds a whole line in shared memory).  The same line limits hold for the slab passes below. */
int nbk_r2c(const void *real, void *cplx, int dtype, const int64_t *nmesh_host, double extra_scale,
            void *stream); /* cplx = extra_scale * FFT(real) / prod(N): folds e.g. the 1/nbar of catalog.py:394-398 */
int nbk_c2r(const void *cplx, void *real, int dtype, const int64_t *nmesh_host, void *work,
            void *stream);

/* Mixed-radix transforms for sides that are products of 2, 3, 5 and 7 (pmesh/pfft accept any size; nbodykit scripts use
 * meshes like 96, 100, 360, 768, 1536): the same RealField.r2c / ComplexField.c2r (base/mesh.py:228,237;
 * source/mesh/catalog.py:341-351) with the semantics of nbk_r2c / nbk_c2r -- forward normalised by 1/(Nx*Ny*Nz) times
 * extra_scale (folded into the last pass), backward unnormalised, c2r preserves its input when `work` is given.
 * Limits: Nx, Ny in 2 .. 4096; Nz in 2 .. 8192 if even, up to 4095 if odd (every complex line <= 4096 points).
 * Powers of two are accepted as well. */
int nbk_r2c_mixed(const void *real, void *cplx, int dtype, const int64_t *nmesh_host, double extra_scale, void *stream);
int nbk_c2r_mixed(const void *cplx, void *real, int dtype, const int64_t *nmesh_host, void *work, void *stream);
/* the passes of the mixed-radix transform, for the slab-decomposed route (P > 1, base/mesh.py:228,237):
 *   lines : complex FFT of length n_line (2 .. 4096, 7-smooth) along element(outer, n, inner) =
 *           data[outer*outer_stride + n*line_stride + inner], inner < n_inner; out = scale * DFT (inverse != 0: the
 *           unnormalised inverse DFT times scale).  src == dst: in place.
 *   z     : real rows [rows][Nz] -> complex rows [rows][Nz/2+1] (inverse == 0), or back (inverse != 0, unnormalised);
 *           the output is multiplied by scale. */
int nbk_fft_lines_mixed(const void *src, void *dst, int dtype, int64_t n_line, int64_t line_stride, int64_t n_inner,
                        int64_t n_outer, int64_t outer_stride, int inverse, double scale, void *stream);
int nbk_fft_z_mixed(const void *in, void *out, int dtype, int64_t rows, int64_t Nz, int inverse, double scale,
                    void *stream);
/* Bluestein (chirp-z) passes with the arguments and semantics of the mixed-radix pair above, for sides with a prime
 * factor above 7 (a cyclic convolution of length M >= 2n - 1, M 7-smooth, done by the mixed-radix stages).  They take
 * any length within the same limits, 7-smooth lengths included: lines 2 .. 4096; Nz even up to 8192, odd up to 4095. */
int nbk_fft_lines_bluestein(const void *src, void *dst, int dtype, int64_t n_line, int64_t line_stride, int64_t n_inner,
                            int64_t n_outer, int64_t outer_stride, int inverse, double scale, void *stream);
int nbk_fft_z_bluestein(const void *in, void *out, int dtype, int64_t rows, int64_t Nz, int inverse, double scale,
                        void *stream);

/* the three 1-D passes of the slab-decomposed transform, for the multi-GPU path (P > 1):
 *   zy pass : real slab [x_n][Ny][Nz] -> cplx slab [x_n][Ny][Nzc], r2c along z then FFT along y
 *   pack    : cplx slab [x_n][Ny][Nzc] -> send buffer [P][y_n][x_n][Nzc] (block p = y rows of rank p)
 *   x pass  : after the all-to-all the receive buffer [P][y_n][x_n][Nzc] IS [y_n][Nx][Nzc] re-ordered;
 *             unpack -> [y_n][Nx][Nzc], FFT along x, scale by `scale`.
 * and their inverses for c2r.
 * nbk_fft_zy_forward (and so nbk_r2c) runs the z and y passes as one pipelined kernel for f8 fields with Nz and Ny in
 * {256, 512, 1024} whose slab is larger than half the L2 (DESIGN 4.2).  Its CTAs coordinate through a ticket counter and progress flags owned by the calling stream:
 * calls on different streams may run concurrently, calls on one stream run in order.  It is not meant for capture into
 * a CUDA graph (a replay would reuse the captured call's flags). */
int nbk_fft_zy_forward(const void *real, void *cplx, int dtype, int64_t x_n, int64_t Ny, int64_t Nz,
                       void *stream);
int nbk_fft_zy_backward(void *cplx, void *real, int dtype, int64_t x_n, int64_t Ny, int64_t Nz,
                        void *stream);
int nbk_fft_lines(void *cplx, int dtype, int64_t n_line, int64_t line_stride, int64_t n_inner,
                  int64_t n_outer, int64_t outer_stride, int inverse, double scale, void *stream);
int nbk_fft_lines_oop(const void *src, void *dst, int dtype, int64_t n_line, int64_t line_stride, int64_t n_inner,
                      int64_t n_outer, int64_t outer_stride, int inverse, double scale, void *stream);
int nbk_fft_z_forward(const void *real, void *cplx, int dtype, int64_t rows, int64_t Nz, void *stream);
int nbk_transpose_pack(const void *src, void *dst, int dtype, int64_t x_n, int64_t Ny, int64_t Nzc,
                       int64_t P, void *stream);
int nbk_transpose_unpack(const void *src, void *dst, int dtype, int64_t y_n, int64_t Nx,
                         int64_t Nzc, int64_t P, void *stream);
int nbk_transpose_pack_back(const void *src, void *dst, int dtype, int64_t y_n, int64_t Nx,
                            int64_t Nzc, int64_t P, void *stream);
int nbk_transpose_unpack_back(const void *src, void *dst, int dtype, int64_t x_n, int64_t Ny,
                              int64_t Nzc, int64_t P, void *stream);

/* Field.apply(func=Compensate*, kind='circular', out=Ellipsis) -- base/mesh.py:306-313 with
 * source/mesh/catalog.py:449-594.  In place on a complex slab. */
int nbk_compensate(void *cplx, int dtype, int kind, const int64_t *nmesh_host, int transposed,
                   int64_t start, int64_t count, void *stream);

/* s1 = 0.5*s1 + 0.5*s2*exp(0.5j * sum_i k_i H_i) -- source/mesh/catalog.py:345-347 */
int nbk_interlace_combine(void *c1, const void *c2, int dtype, const int64_t *nmesh_host,
                          const double *boxsize_host, int transposed, int64_t start, int64_t count,
                          void *stream);

/* FFTBase._compute_3d_power (algorithms/fftpower.py:115-128: c1*conj(c2), zero mode, *V) fused
 * with project_to_basis (:507-701) and MeshSlab.norm2/mu/hermitian_weights (meshtools.py:104-215).
 * c2 == NULL -> auto power.  If is_p3d != 0 the input is taken as an already-formed 3-D statistic
 * y3d (project_to_basis semantics only; c2, volume, clear_zero ignored).
 * k2edges: host double[Nx+1] = kedges**2; muedges: host double[Nmu+1]; ells: host int[Nell]
 * (ells[0] must be 0).  coord_dtype NBK_F4 (fixture-faithful) | NBK_F8.
 * comp1 / comp2 (NBK_COMP_*): window compensation applied on the fly to c1 / c2 (the fused equivalent of
 * running nbk_compensate on each field first); NBK_COMP_NONE when the fields are already compensated.
 * hermitian: 0 full field, 1 Hermitian-compressed last axis with y(-k) = conj y(k), 2 compressed with
 * y(-k) = -conj y(k) (the odd multipoles of ConvolvedFFTPower, A0 conj(A_l): what the reference obtains from a full
 * 'c16' mesh, convpower/catalog.py:169-176); the mirror half is folded in accordingly.
 * real_input != 0: c1 is a REAL [count][D1][Nz] statistic (FFTCorr, algorithms/fftcorr.py:148-176; needs is_p3d,
 * hermitian == 0).  coord_unit_host: per-axis coordinate of index 1 (NULL -> 2 pi / L, the wavenumbers; FFTCorr
 * passes the cell size L/N so that coordinates are the wrapped separations).
 * Outputs (device, ACCUMULATED into; zero first), nb = (Nx+2)*(Nmu+2):
 *   nsum int64[nb]; xsum, musum double[nb]; ysum double[Nell][nb][2] (re, im).  * musum may be NULL when the caller never reads the per-bin sum of mu (FFTPower mode='1d'): that reduction is then skipped. */
int nbk_power_bin(const void *c1, const void *c2, int dtype, int is_p3d, double volume,
                  int clear_zero, const int64_t *nmesh_host, const double *boxsize_host,
                  int transposed, int64_t start, int64_t count, int coord_dtype,
                  const double *k2edges_host, int Nx, const double *muedges_host, int Nmu,
                  const double *los_host, const int *ells_host, int Nell, int hermitian, int comp1,
                  int comp2, int real_input, const double *coord_unit_host, int64_t *nsum, double *xsum, double *musum, double *ysum, void *stream);

/* The last pass of nbk_r2c fused with the FFTPower mode '1d' auto power of nbk_power_bin, for one rank: cplx holds the
 * whole Hermitian-compressed mesh after nbk_fft_zy_forward.  Runs the x pass scaled by extra_scale / (Nx*Ny*Nz) and
 * bins each mode as nbk_power_bin(c1 = cplx, c2 = NULL, is_p3d = 0, clear_zero = 1, coord_dtype = 4, ells = {0},
 * hermitian = 1, comp1 = comp2 = comp, musum = NULL) would bin the transformed field, without storing it: cplx is left
 * as it was.  Outputs as nbk_power_bin's (nb = (Nx+2)*3, accumulated into; the imaginary parts are not touched).
 * *fused = 0: the case does not take the fused kernel (f4 fields, line of sight not along z, mu edges other than
 * {-1, 1}, Nx not in {256, 512, 1024}, too many k bins for shared memory); nothing ran, and the caller runs the x pass with nbk_fft_lines
 * and then nbk_power_bin. */
int nbk_fft_x_power_bin(void *cplx, int dtype, const int64_t *nmesh_host, const double *boxsize_host,
                        double extra_scale, double volume, const double *k2edges_host, int Nx,
                        const double *muedges_host, int Nmu, const double *los_host, int comp, int64_t *nsum,
                        double *xsum, double *ysum, int *fused, void *stream);

/* nbk_power_bin with a third field: c2_mirror stands for c2 at the UNSTORED mirror mode -k of every mode with
 * 0 < j_z < N_z/2, i.e. the mirror's share of the sum is conj(c1 conj(c2_mirror)) V instead of the (anti-)Hermitian
 * fold of c1 conj(c2).  This is what a full complex ('c16') mesh gives the reference when c2 carries a factor that is
 * not parity-symmetric on the Nyquist planes -- A_l = sum_m Y_lm(khat) FFT[F Y_lm] of ConvolvedFFTPower
 * (algorithms/convpower/fkp.py:571-623; convpower/catalog.py:169-176): the mirror of index N/2 keeps the label -N/2
 * (meshtools.py:150-153), so Y_lm(khat) at the mirror is not (-1)^l Y_lm(khat).  hermitian must be 1. */
int nbk_power_bin2(const void *c1, const void *c2, const void *c2_mirror, int dtype, int is_p3d, double volume,
                   int clear_zero, const int64_t *nmesh_host, const double *boxsize_host,
                   int transposed, int64_t start, int64_t count, int coord_dtype,
                   const double *k2edges_host, int Nx, const double *muedges_host, int Nmu,
                   const double *los_host, const int *ells_host, int Nell, int hermitian, int comp1,
                   int comp2, int real_input, const double *coord_unit_host, int64_t *nsum, double *xsum, double *musum, double *ysum, void *stream);

/* out = c1 * conj(c2) * scale with element 0 cleared when clear_first != 0 (the k = 0 mode on the rank that owns
 * it): FFTBase._compute_3d_power (algorithms/fftpower.py:115-128), materialised only where the 3-D power itself
 * is needed (FFTCorr, algorithms/fftcorr.py:148-150; FFT3PCF's kernel products).  c2 == NULL -> auto power.  out may
 * alias c1 or c2: every element's inputs are read before that element is written. */
int nbk_cross_power(const void *c1, const void *c2, void *out, int dtype, int64_t n_complex, double scale,
                    int clear_first, void *stream);

/* ConvolvedFFTPower's spherical-harmonic passes (algorithms/convpower/fkp.py:571-597), real Y_lm, l <= 8:
 *   out(x) = in(x) * Y_lm(xhat), x = wrapped grid coordinate [-L/2, L/2) + offset[3] (BoxCenter + H/2, :457);
 *   acc(k) += c(k) * Y_lm(khat), khat := 0 at k = 0 (:537). */
int nbk_ylm_mul_real(const void *in, void *out, int dtype, int l, int m, const int64_t *nmesh_host,
                     const double *boxsize_host, const double *offset_host, int64_t x_start, int64_t x_n,
                     void *stream);
int nbk_ylm_mul_complex_acc(void *acc, const void *c, int dtype, int l, int m, const int64_t *nmesh_host,
                            const double *boxsize_host, int transposed, int64_t start, int64_t count,
                            void *stream);

/* nbk_ylm_mul_complex_acc plus a second accumulator evaluated with the direction the mirror mode -k carries on a full
 * complex mesh: every component flips sign except those at the Nyquist index (label stays -N/2) -- the c2_mirror of
 * nbk_power_bin2. */
int nbk_ylm_mul_complex_acc2(void *acc, void *acc_mirror, const void *c, int dtype, int l, int m,
                             const int64_t *nmesh_host, const double *boxsize_host, int transposed, int64_t start,
                             int64_t count, void *stream);

/* Complex-dtype meshes (ParticleMesh(dtype='c16'/'c8'), base/mesh.py:50; convpower/catalog.py:151-176): pmesh keeps all
 * N^3 modes of the c2c transform.  The configuration-space fields of this path are real-valued, so the full spectrum
 * is the Hermitian completion of the r2c result: full[Nx][Ny][Nz] <- comp[Nx][Ny][Nz/2+1] (single GPU), and the
 * stored half is cut back out before a c2r (rows = planes * Ny of this rank). */
int nbk_hermitian_expand(const void *comp, void *full, int dtype, const int64_t *nmesh_host, void *stream);
int nbk_hermitian_compress(const void *full, void *comp, int dtype, int64_t rows, int64_t Nz, void *stream);

/* Slab transpose over NVLink peer memory for the pencil transpose of pfft (r2c / c2r, base/mesh.py:228,237): a line
 * pass (FFT along the second stored axis of src[n_outer][n_line][n_inner]) into P contiguous local send blocks
 * send[p][k % (N/P)][n_outer][inner], followed by one strided bulk copy per peer (cudaMemcpy2DAsync, rows of
 * n_outer * n_inner elements).  nbk_slab_push_range: block p of `send` -> rank p's field
 * [rows_per_peer][n_outer * P][n_inner] at offset outer_start; peer_ptrs_host: host array of P device pointers valid
 * on this GPU (entry `rank` = the local buffer).  Both steps cover the outer sub-range [o0, o0 + o_cnt) of the slab
 * (planes of x in r2c, base/mesh.py:237): the caller pushes one part on a second stream while the line pass of the
 * next part runs; o0 = 0, o_cnt = n_outer is the whole slab.  The caller provides the cross-rank barriers. */
int nbk_fft_lines_pack_range(const void *src, void *send, int dtype, int64_t n_line, int64_t n_inner, int64_t n_outer,
                             int64_t o0, int64_t o_cnt, int P, int inverse, double scale, void *stream);
int nbk_slab_push_range(const void *send, void *const *peer_ptrs_host, int dtype, int64_t rows_per_peer, int64_t n_outer,
                        int64_t n_inner, int64_t outer_start, int64_t o0, int64_t o_cnt, int P, int rank, void *stream);

/* Fourier-space resampling to another mesh size: pmesh `Field.resample`, called by MeshSource.compute(Nmesh=...)
 * (base/mesh.py:317-327).  Per axis, destination index i has the label j = i < (N+1)/2 ? i : i - N and is copied from
 * the source mode with the same label when -m <= 2j < m, m = min(N_src, N_dst) (even m: the Nyquist label is negative);
 * along the compressed z axis indices 0 .. m/2 map to themselves.  Everything else in dst is zero.  Any sides 2 .. 2^24-1.
 * Hermitian-compressed single-GPU layouts [Nx][Ny][Nz/2+1]. */
int nbk_resample_complex(const void *src, void *dst, int dtype, const int64_t *nmesh_src_host,
                         const int64_t *nmesh_dst_host, void *stream);
/* The same rule on P > 1, where each rank holds the transposed slab [y_n][Nx][Nz/2+1] of both meshes.  The caller plans
 * which y rows travel between which ranks and passes them as `n_ranges` (<= 32) pairs ranges_host[2i] = first local row,
 * ranges_host[2i+1] = count, in send (pack) or receive (unpack) order; one all-to-all moves the send blocks.
 *   pack   : send [rows listed][Nx_dst][Nz_dst/2+1] <- the listed rows of src [src_rows][Nx_src][Nz_src/2+1], remapped
 *            in x and z.
 *   unpack : dst [dst_rows][Nx_dst][Nz_dst/2+1]: the listed rows <- recv in order (ranges must not overlap), every
 *            other row zero. */
int nbk_resample_pack(const void *src, void *send, int dtype, const int64_t *nmesh_src_host, const int64_t *nmesh_dst_host,
                      int64_t src_rows, const int64_t *ranges_host, int n_ranges, void *stream);
int nbk_resample_unpack(const void *recv, void *dst, int dtype, const int64_t *nmesh_dst_host, int64_t dst_rows,
                        const int64_t *ranges_host, int n_ranges, void *stream);

/* Friends-of-friends groups (algorithms/fof.py: `_fof_local`, `_fof_merge`, `_assign_labels`, `centerofmass`,
 * `fof_catalog`).  Two particles are friends when d^2 = (dx^2 + dy^2) + dz^2 <= b^2, evaluated in double from the stored
 * positions (no FMA); periodic: positions wrapped as numpy's `pos % L` in their own dtype, per-axis |d| -> min(|d|, L - |d|).
 * Rows: n < 2^32.  The cell grid has ncell_host[d] cells of side box[d] / ncell[d] <= b / sqrt(3) per axis (non-periodic:
 * starting at origin_host, box = extent); cells are 63-bit keys (x-major).
 *   cell_keys   : keys[n] (int64) of every particle.
 *   sort        : stable LSD radix sort of `keys` (uint64, key_bytes 8, or uint32, key_bytes 4; bits [0, end_bit)) carrying
 *                 the row index (uint32, filled by the call) along; n < 2^31.  keys/keys_alt and rows/rows_alt are the two
 *                 halves of a double buffer; *result_in_alt (host) says which one holds the result.  work: device scratch
 *                 of nbk_fof_sort_workspace(n, key_bytes) bytes.
 *   sorted_pos  : sorted_pos[i] = (wrapped) pos[perm[i]], perm = the key sort permutation (uint32).
 *   compact     : occupied cells of the sorted keys.  compact_count: *ncells (device int64); compact_write:
 *                 cell_start[0..ncells] (uint32, last entry = n), cell_key[ncells].  work: device
 *                 int64[nbk_fof_compact_workspace(n)], the same for both calls.
 *   link        : union-find over the cells: parent[ncells] (uint32, every entry its root on return), cell_min[ncells] (smallest
 *                 global id in the cell; at a root, of its component).  Global id of row r: gid[r], or gid_base + r when gid is
 *                 NULL.  Every pair of cells within reach is united when one particle pair links.
 *   finalize    : per row r: row_root[r] = root cell, minid[r] = smallest global id of its group (minid may be NULL).
 *   lower       : per row, minid[r] <- the smallest new_minid[] over the rows of its root (the `_fof_merge` step on one rank);
 *                 *changed (device uint64, accumulated) += rows whose value changed.  root_min: device int64[ncells] scratch.
 *   root_counts : counts[row_root[r]] += 1 (device uint64[ncells], zero first).
 *   label_rows  : labels[r] = cell_label[row_root[r]] as int32 (label_bytes 4) or int64 (8).
 *   segment_reduce : rows ordered by label (`order`, uint32), split into chunks: chunk k = sorted rows [chunk_first[k], chunk_first[k+1])
 *                 of label chunk_label[k]; label l owns chunks [label_chunk[l], label_chunk[l+1]).  Fixed-order reduction into
 *                 out[nlabels][4] (partial: device double[nchunks][4] scratch):
 *                   NBK_FOF_RED_MIN  per-axis minimum of a [n][3] column        (slot 3: rows)
 *                   NBK_FOF_RED_MAX  maximum of a [n] column in slot 0          (slot 3: rows)
 *                   NBK_FOF_RED_SUM  per-axis sum of col - ref[l] (ref NULL: col), wrapped into [-L/2, L/2) when periodic
 *                                    and ref is given; slot 3: rows
 *                 mask != NULL restricts MIN / SUM to rows with mask[r] >= thresh[l]. */
#define NBK_FOF_RED_MIN 0
#define NBK_FOF_RED_MAX 1
#define NBK_FOF_RED_SUM 2
int nbk_fof_cell_keys(const void *pos, int pos_dtype, int64_t n, int periodic, const double *box_host,
                      const double *origin_host, const int64_t *ncell_host, double b, int64_t *keys, void *stream);
/*   grid_keys   : the keys of cell_keys on a grid of any cell size (no linking length; used by the pair counts). */
int nbk_fof_grid_keys(const void *pos, int pos_dtype, int64_t n, int periodic, const double *box_host,
                      const double *origin_host, const int64_t *ncell_host, int64_t *keys, void *stream);
int64_t nbk_fof_sort_workspace(int64_t n, int key_bytes);
int nbk_fof_sort(void *keys, void *keys_alt, uint32_t *rows, uint32_t *rows_alt, int64_t n, int key_bytes, int end_bit,
                 void *work, int64_t work_bytes, int *result_in_alt, void *stream);
int nbk_fof_sorted_pos(const void *pos, int pos_dtype, int64_t n, const uint32_t *perm, int periodic,
                       const double *box_host, void *sorted_pos, void *stream);
int64_t nbk_fof_compact_workspace(int64_t n);
int nbk_fof_compact_count(const int64_t *sorted_keys, int64_t n, int64_t *work, int64_t work_len, int64_t *ncells,
                          void *stream);
int nbk_fof_compact_write(const int64_t *sorted_keys, int64_t n, const int64_t *work, int64_t work_len,
                          uint32_t *cell_start, int64_t *cell_key, void *stream);
int nbk_fof_link(const void *sorted_pos, int pos_dtype, const uint32_t *perm, const int64_t *gid, int64_t gid_base,
                 const uint32_t *cell_start, const int64_t *cell_key, int64_t ncells, int periodic, const double *box_host,
                 const double *origin_host, const int64_t *ncell_host, double b, uint32_t *parent, int64_t *cell_min,
                 void *stream);
int nbk_fof_finalize(const uint32_t *perm, const uint32_t *cell_start, int64_t ncells, const uint32_t *parent,
                     const int64_t *cell_min, uint32_t *row_root, int64_t *minid, void *stream);
int nbk_fof_lower(const uint32_t *row_root, int64_t n, const int64_t *new_minid, int64_t ncells, int64_t *root_min,
                  int64_t *minid, uint64_t *changed, void *stream);
int nbk_fof_root_counts(const uint32_t *row_root, int64_t n, uint64_t *counts, void *stream);
int nbk_fof_label_rows(const uint32_t *row_root, int64_t n, const int64_t *cell_label, void *labels, int label_bytes,
                       void *stream);
int nbk_fof_segment_reduce(int op, const void *col, int col_dtype, const void *mask, int mask_dtype, const double *thresh,
                           const double *ref, int periodic, const double *box_host, const uint32_t *order,
                           const int64_t *chunk_first, const int64_t *chunk_label, int64_t nchunks,
                           const int64_t *label_chunk, int64_t nlabels, double *partial, double *out, void *stream);

/* Binned pair counts in a simulation box or a survey (algorithms/paircount.py: SimulationBoxPairCount,
 * algorithms/surveypaircount.py: SurveyDataPairCount; DESIGN.md 4.6, 4.8).  Positions are double [n][3] with the line
 * of sight in the last column (periodic: already wrapped), both catalogues key-sorted on the same grid of
 * ncell_host[d] cells of side box[d] / ncell[d] (nbk_fof_grid_keys / sort / compact / sorted_pos).
 * Primary chunk k = sorted primary rows [chunk_first[k], chunk_first[k+1]), at most nbk_paircount_chunk_rows() rows of
 * the one cell chunk_key[k].  Secondaries: spos / sw sorted, cell table scell_start[nscells + 1] / scell_key[nscells].
 * tol_host[d]: how far a row may lie outside its cell (cells are skipped only when every pair is out of range by more).
 * mode NBK_PC_1D: bins of s over `edges`; NBK_PC_2D: (s, mu = |dc| / s) over edges x edges2 (mu = 1 in the last bin);
 * NBK_PC_PROJECTED: (r_p, |dc|) over edges x edges2 for |dc| < pimax.  Bin k of `edges` holds e_k^2 <= x^2 < e_{k+1}^2
 * (squares taken here in double).  The survey modes (periodic must be 0) take the observer at the origin and the
 * pair's midpoint as its line of sight: s = x2 - x1, l = x1 + x2 per axis, l^2 = (lx^2 + ly^2) + lz^2,
 * sl = (sx lx + sy ly) + sz lz.  NBK_PC_SURVEY_2D: (s, mu = |sl| / (s sqrt(l^2)), 0 when l^2 = 0) as NBK_PC_2D;
 * NBK_PC_SURVEY_PROJECTED: pi = |sl| / sqrt(l^2) (0 when l^2 = 0), r_p^2 = max(s^2 - pi^2, 0), (r_p, pi) as
 * NBK_PC_PROJECTED for pi < pimax; NBK_PC_ANGULAR: unit vectors, `edges` are chords 2 sin(theta / 2), bins of the chord
 * as NBK_PC_1D, summing theta = 2 asin(chord / 2) in degrees.  Accumulates (device, zero first) npairs[nbins]
 * (uint64), wsum[nbins] (sum of pw * sw) and ssum[nbins] (sum of s, r_p or theta), and *candidates (uint64) += pairs
 * tested.  work: device double scratch of len(edges) + len(edges2) (1d / angular: + 2) entries.  Histograms above
 * nbk_paircount_smem_bins() bins take global atomics. */
#define NBK_PC_1D 1
#define NBK_PC_2D 2
#define NBK_PC_PROJECTED 3
#define NBK_PC_SURVEY_2D 4
#define NBK_PC_SURVEY_PROJECTED 5
#define NBK_PC_ANGULAR 6
int64_t nbk_paircount_chunk_rows(void);
int64_t nbk_paircount_smem_bins(void);
int nbk_paircount(int mode, const double *ppos, const double *pw, const int64_t *chunk_first, const int64_t *chunk_key,
                  int64_t nchunks, const double *spos, const double *sw, const uint32_t *scell_start, const int64_t *scell_key,
                  int64_t nscells, int periodic, const double *box_host, const int64_t *ncell_host, const double *tol_host,
                  const double *edges_host, int nedges, const double *edges2_host, int nedges2, double pimax, double *work,
                  uint64_t *npairs, double *wsum, double *ssum, uint64_t *candidates, void *stream);

/* Multipoles of the isotropic three-point function in a simulation box (algorithms/threeptcf.py: SimulationBox3PCF;
 * DESIGN.md 4.7).  Positions, chunks and the secondary cell table as for nbk_paircount (chunks of at most
 * nbk_threeptcf_chunk_rows() primaries of one cell; no line-of-sight reordering).  Per axis d = x_j - x_p in double
 * (periodic: d > L/2 -> d - L, d <= -L/2 -> d + L), r = sqrt((dx^2 + dy^2) + dz^2); radial bin k of `edges` (e_0 >= 0,
 * at most nbk_threeptcf_max_bins() bins) holds e_k < r <= e_{k+1}, r > 0.  poles_host: npoles distinct l in
 * 0 .. nbk_threeptcf_max_ell(); L = max l.  coef_host: [(L+1)(L+2)/2][L+1] table T with a_lm = sum_k T[lm][k] M_{m,k},
 * lm = off(m) + l - m, off(m) = m (L + 1) - m (m - 1) / 2, M_{m,k}(b) = sum_{j in b} w_j (ux + i uy)^m uz^k.
 * Accumulates (device, zero first) zeta[npoles][nb][nb] (b1 <= b2 only) += sum_p w_p sum_m c_m Re[a_lm(b1) a*_lm(b2)]
 * with c_0 = 1, c_m = 2 (m > 0), npairs[nb] (uint64, ordered (p, j) pairs per bin) and *candidates += pairs tested.
 * work: device double scratch of nedges + (L+1)^2 (L+2) / 2 entries. */
int64_t nbk_threeptcf_chunk_rows(void);
int nbk_threeptcf_max_ell(void);
int nbk_threeptcf_max_bins(void);
int nbk_threeptcf(const double *ppos, const double *pw, const int64_t *chunk_first, const int64_t *chunk_key, int64_t nchunks,
                  const double *spos, const double *sw, const uint32_t *scell_start, const int64_t *scell_key, int64_t nscells,
                  int periodic, const double *box_host, const int64_t *ncell_host, const double *tol_host, const double *edges_host,
                  int nedges, const int *poles_host, int npoles, const double *coef_host, double *work, double *zeta,
                  uint64_t *npairs, uint64_t *candidates, void *stream);

/* FFT bispectrum of a periodic box (algorithms/bispectrum.py: FFTBispectrum; DESIGN.md 4.14).  At most
 * nbk_bispec_max_shells() k shells.
 *   fill       : one pass over the Hermitian-compressed Fourier slab cplx (layout / start / count as nbk_power_bin takes
 *                them; NBK_LAYOUT_FULLZ is refused) writes shells [shell0, shell0 + nshell) of the nedges - 1 shells of
 *                k2edges_host (squared k edges): out[s][slab] = c * 1_S (complex of dtype) or, indicator != 0, the
 *                complex f8 indicator 1_S, s = 0 .. nshell - 1, out_stride complex elements apart.  A mode is in shell
 *                b - 1 when nbk_power_bin puts it in bin b at float32 coordinates; the k = 0 mode is in no shell.
 *   fill_poles : the same pass writes, for the nell even multipoles ells_host[q] (0 .. 8, at most 5) and the same shells,
 *                out[q nshell + s][slab] = c * L_ell(mu) * 1_S (complex of dtype), out_stride complex elements apart;
 *                mu = k.los / |k| in float32 as nbk_power_bin forms it for a Python-number los (coordinate mode 4),
 *                L_ell in float64, the product rounded once to dtype.
 *   fill_cross : the same pass over two slabs cplx, cplx2 of the same layout and dtype writes, for the same shells,
 *                out[s][slab] = scale * c * conj(c2) * 1_S as complex f8 (the product formed in float64), out_stride
 *                complex elements apart.
 *   triple_sum : fields holds nfield real fields of ncell values (dtype), field_stride elements apart; triples ntri
 *                device int triples (i, j, l) of slots < nfield.  Accumulates (device, zero first)
 *                out[t] += sum_x f_i f_j f_l, products and sums in float64. */
int nbk_bispec_max_shells(void);
int nbk_bispec_fill(const void *cplx, int dtype, const int64_t *nmesh_host, const double *box_host, int layout, int64_t start,
                    int64_t count, const double *k2edges_host, int nedges, int shell0, int nshell, int indicator, void *out,
                    int64_t out_stride, void *stream);
int nbk_bispec_fill_poles(const void *cplx, int dtype, const int64_t *nmesh_host, const double *box_host, int layout,
                          int64_t start, int64_t count, const double *k2edges_host, int nedges, int shell0, int nshell,
                          const double *los_host, const int *ells_host, int nell, void *out, int64_t out_stride, void *stream);
int nbk_bispec_fill_cross(const void *cplx, const void *cplx2, int dtype, const int64_t *nmesh_host, const double *box_host,
                          int layout, int64_t start, int64_t count, const double *k2edges_host, int nedges, int shell0,
                          int nshell, double scale, void *out, int64_t out_stride, void *stream);
int nbk_bispec_triple_sum(const void *fields, int dtype, int64_t field_stride, int nfield, int64_t ncell, const int *triples,
                          int64_t ntri, double *out, void *stream);

/* FFT three-point correlation function of a periodic box (algorithms/fft3pcf.py: FFT3PCF; DESIGN.md 4.16).
 *   kernel_fill : on the local x slab [x_start, x_start + x_n) of a real mesh (layout [x_n][Ny][Nz], dtype), writes for
 *                 the real orthonormal harmonics m = m0 .. m0 + nm - 1 of multipole ell (m > 0: sqrt(2) Re Y_lm, m < 0:
 *                 sqrt(2) Im Y_l|m|) the fields out[q][slab] = Y_l(m0+q)(s / r) at the cells whose grid separation s =
 *                 (n_x H_x, n_y H_y, n_z H_z), n_i in (-N_i/2, N_i/2], H_i = box_i / N_i, has edges[bin] < r <= edges[bin
 *                 + 1] and r > 0, r = sqrt((sx^2 + sy^2) + sz^2) in float64; 0 at every other cell; out_stride elements
 *                 apart.  coef_host is SimulationBox3PCF's coefficient_table(L) ((L + 1)(L + 2) / 2 rows of L + 1,
 *                 ell <= L <= 10); Y_lm is evaluated in float64 and rounded once to dtype.
 *   gram        : w, A and B are real fields of ncell values (dtype); A holds na fields a_stride apart, B nb fields
 *                 b_stride apart (1 .. 32 each).  Accumulates (device, zero first) out[i][j] +=
 *                 sum_x w a_i b_j, row-major na x nb, products and sums in float64.  When B is A (same pointer, count
 *                 and stride) only the entries i <= j are added.
 *   gram_tiles  : gram over the cells of the tiles tiles[0 .. ntiles) only (device int64, each in [0, ceil(ncell / 64)),
 *                 tile t = cells 64 t .. 64 t + 63); w must be 0 on every cell of the tiles left out, so the sum is
 *                 gram's up to summation order (algorithms/convfft3pcf.py: ConvolvedFFT3PCF; DESIGN.md 4.17). */
int nbk_fft3pcf_kernel_fill(void *out, int dtype, const int64_t *nmesh_host, const double *box_host, int64_t x_start,
                            int64_t x_n, const double *edges_host, int nedges, int bin, int ell, int m0, int nm,
                            const double *coef_host, int L, int64_t out_stride, void *stream);
int nbk_fft3pcf_gram(const void *w, const void *A, int64_t a_stride, int na, const void *B, int64_t b_stride, int nb,
                     int dtype, int64_t ncell, double *out, void *stream);
int nbk_fft3pcf_gram_tiles(const void *w, const void *A, int64_t a_stride, int na, const void *B, int64_t b_stride,
                           int nb, int dtype, int64_t ncell, const int64_t *tiles, int64_t ntiles, double *out,
                           void *stream);

/* Cylindrical groups (algorithms/cgm.py: CylindricalGroups; DESIGN.md 4.9).  Rows key-sorted on a grid of ncell_host[d]
 * cells of side box[d] / ncell[d] as for nbk_paircount: spos double [n][3] (periodic: already wrapped), sprio[n] the
 * distinct global priority of each sorted row, perm[n] its row before sorting; rows with perm < n_own are owned, the
 * others are copies.  Chunks of at most nbk_cgm_chunk_rows() sorted rows of one cell.  Rows a != b (a the higher
 * priority) are linked iff |dr2 - rlos2| <= rperp^2 and rlos2 <= rpar^2, dr = x_a - x_b (periodic: minimum image with
 * dr > L/2 -> dr - L, dr <= -L/2 -> dr + L), dr2 = (dx^2 + dy^2) + dz^2; los_host (a 3-vector): rlos2 = t^2 with
 * t = (dx lx + dy ly) + dz lz; los_host NULL: c = (x_a + x_b) / 2, rlos2 = ((dx cx + dy cy) + dz cz)^2 / |c|^2 and no
 * link when |c|^2 = 0.  Everything in double.
 *   count  : counts[i] = higher-priority rows linked to owned sorted row i (copies: untouched); *candidates += pairs tested
 *   write  : their sorted row indices at nbr[offsets[i] ..] (offsets: exclusive scan of counts, n + 1 entries)
 *   resolve: one round over order[n_own] (owned sorted rows, descending priority) of state (0 undecided, 1 central,
 *            2 satellite, per sorted row): undecided rows with a central neighbour become satellites, those whose
 *            neighbours are all satellites (or none) centrals; *undecided += owned rows left undecided
 *   assign : cen_prio[r] = the priority of the central of owned row r (its own for a central), nsat[central] += 1 per
 *            satellite (uint64, per sorted row, zero first). */
int64_t nbk_cgm_chunk_rows(void);
int nbk_cgm_count(const double *spos, const int64_t *sprio, const uint32_t *perm, int64_t n, int64_t n_own,
                  const int64_t *chunk_first, const int64_t *chunk_key, int64_t nchunks, const uint32_t *cell_start,
                  const int64_t *cell_key, int64_t ncells, int periodic, const double *box_host, const int64_t *ncell_host,
                  const double *tol_host, const double *los_host, double rperp, double rpar, int64_t *counts,
                  uint64_t *candidates, void *stream);
int nbk_cgm_write(const double *spos, const int64_t *sprio, const uint32_t *perm, int64_t n, int64_t n_own,
                  const int64_t *chunk_first, const int64_t *chunk_key, int64_t nchunks, const uint32_t *cell_start,
                  const int64_t *cell_key, int64_t ncells, int periodic, const double *box_host, const int64_t *ncell_host,
                  const double *tol_host, const double *los_host, double rperp, double rpar, const int64_t *offsets,
                  int32_t *nbr, void *stream);
int nbk_cgm_resolve(const int32_t *order, int64_t n_own, const int64_t *offsets, const int32_t *nbr, uint8_t *state,
                    uint64_t *undecided, void *stream);
int nbk_cgm_assign(const int32_t *order, int64_t n_own, const int64_t *offsets, const int32_t *nbr, const uint8_t *state,
                   const int64_t *sprio, int64_t *cen_prio, uint64_t *nsat, void *stream);

/* Nearest-neighbour distances in the periodic unit box (algorithms/kdtree.py: KDDensity; DESIGN.md 4.10).  K =
 * nbk_kd_k() (8).  Distance of unit positions a, b in double: dx = a_x - b_x, dx > 0.5 -> dx - 1, dx < -0.5 -> dx + 1 per
 * axis, d2 = (dx^2 + dy^2) + dz^2.
 *   unit      : q (double [n][3]) = pos / L in the positions' dtype (float32: f4(f8(x) / L)), then numpy's q % 1 in that
 *               dtype; a q of 1.0 becomes 0.0
 *   cell_table: dense[k] (ncell[0] ncell[1] ncell[2] + 1 entries) = the first sorted row of cell key k, from the compact
 *               table of nbk_fof_compact_write (cell_start[ncells + 1], cell_key[ncells])
 *   self      : rows key-sorted on the grid of ncell_host[d] cells of side 1 / ncell[d]: spos double [n][3] in [0, 1), perm[n]
 *               the row before sorting; rows with perm < n_own are owned, the others are copies.  kth[perm[i]] = the K-th
 *               smallest d2 from owned sorted row i to all n rows, itself included (+inf with fewer than K rows)
 *   query     : knn[i][0 .. K-1] = the K smallest d2 from qpos[i] (double [nq][3] in [0, 1)) to the owned rows, ascending
 *   density   : dist[i] = sqrt(d2[i]), density[i] = 1 / (dist[i]^3 volume)
 * self and query add the rows they test to *candidates (device uint64). */
int64_t nbk_kd_k(void);
int nbk_kd_unit(const void *pos, int pos_dtype, int64_t n, double L, double *q, void *stream);
int nbk_kd_cell_table(const uint32_t *cell_start, const int64_t *cell_key, int64_t ncells, const int64_t *ncell_host,
                      uint32_t *dense, void *stream);
int nbk_kd_self(const double *spos, const uint32_t *perm, int64_t n, int64_t n_own, const uint32_t *dense,
                const int64_t *ncell_host, double *kth, uint64_t *candidates, void *stream);
int nbk_kd_query(const double *qpos, int64_t nq, const double *spos, const uint32_t *perm, int64_t n, int64_t n_own,
                 const uint32_t *dense, const int64_t *ncell_host, double *knn, uint64_t *candidates, void *stream);
int nbk_kd_density(const double *d2, int64_t n, double volume, double *dist, double *density, void *stream);

/* Fiber collisions (algorithms/fibercollisions.py: FiberCollisions; DESIGN.md 4.11).  The members of the FOF groups of
 * at least 2 rows, sorted by (label, global row): pos float [n][3] (unit-sphere positions + 1.1, cast to float32), grow
 * int64 [n] their global rows, gstart int64 [groups + 1] the first member of every group.  Members a, b collide when
 * sqrt((dx^2 + dy^2) + dz^2) <= rad, in double from the float32 positions.  The greedy of a group removes, among the alive
 * members with the most alive colliders (n_coll) and then the fewest colliders of those colliders (n_other), the
 * ((h >> 32) k) >> 32-th of the k candidates in member order, h = SplitMix64 of (seed, the group's first global row,
 * removals so far); it stops when no alive member has a collider.  collided (int32 [n], zeroed) gets 1 and neighbor (int64
 * [n], -1) the global row of the nearest uncollided member (the first in member order on a tie) of every removed member.
 *   pairs       : the groups gid[0 .. ng-1] of exactly 2 members: the pick of the two, without a distance test
 *   small       : the groups gid[0 .. ng-1] of 3 .. nbk_fc_warp_members() members, one warp each
 *   larger groups q = 0 .. nlg-1: member m of q is l = lbeg[q] + m (lq[l] = q), at segment row lseg[q] + m
 *   cell_keys   : keys[l] of segment row lrow[l] on nc^3 cells of side cs >= rad over [0, nc cs)^3
 *   count/write : counts[l] = colliders of l, then their group-local indices at nbr[offsets[l] ..]; cidx / ckey are the l
 *                 sorted by (q, key) and their keys
 *   greedy      : one block per group; groups above nbk_fc_smem_members() members keep their state in the scratch arrays
 *                 (indexed by l); nunc[q] = members left uncollided
 *   nearest     : the neighbor of every collided member of the larger groups, by a walk over rings of cells
 * small and greedy add their removals to *steps, and count the members it tests to *candidates (device uint64). */
int64_t nbk_fc_warp_members(void);
int64_t nbk_fc_smem_members(void);
int nbk_fc_pairs(const int64_t *gstart, const int32_t *gid, int64_t ng, const int64_t *grow, uint64_t seed, int32_t *collided,
                 int64_t *neighbor, void *stream);
int nbk_fc_small(const float *pos, const int64_t *gstart, const int32_t *gid, int64_t ng, const int64_t *grow, double rad,
                 uint64_t seed, int32_t *collided, int64_t *neighbor, uint64_t *steps, void *stream);
int nbk_fc_cell_keys(const float *pos, const int64_t *lrow, int64_t nl, double cs, int64_t nc, int64_t *keys, void *stream);
int nbk_fc_count(const float *pos, const int32_t *lq, const int64_t *lbeg, const int64_t *lseg, int64_t nl, const int32_t *cidx,
                 const int64_t *ckey, double cs, int64_t nc, double rad, int64_t *counts, uint64_t *candidates, void *stream);
int nbk_fc_write(const float *pos, const int32_t *lq, const int64_t *lbeg, const int64_t *lseg, int64_t nl, const int32_t *cidx,
                 const int64_t *ckey, double cs, int64_t nc, double rad, const int64_t *offsets, int32_t *nbr, void *stream);
int nbk_fc_greedy(const int64_t *lbeg, const int64_t *lseg, int64_t nlg, int64_t max_members, const int64_t *offsets,
                  const int32_t *nbr, const int64_t *grow, uint64_t seed, int32_t *scratch_ncoll, int64_t *scratch_nother,
                  uint8_t *scratch_alive, int32_t *collided, int64_t *nunc, uint64_t *steps, void *stream);
int nbk_fc_nearest(const float *pos, const int32_t *lq, const int64_t *lbeg, const int64_t *lseg, int64_t nl, const int32_t *cidx,
                   const int64_t *ckey, double cs, int64_t nc, const int32_t *collided, const int64_t *nunc, const int64_t *grow,
                   int64_t *neighbor, void *stream);

/* Redshift histogram n(z) (algorithms/zhist.py: RedshiftHistogram; DESIGN.md 4.12).  z (and w) are float32 or float64
 * (NBK_F4 / NBK_F8), widened exactly to double; n rows, 64-bit.
 *   moments : out[6] (device double) = count, mean, M2 (sum of squared deviations from the mean), min and max of the
 *             finite rows, and the number of non-finite rows.  partial: device scratch of nbk_zh_partials() * 6 doubles.
 *             The merge order depends on n alone: the same rows give the same bits on every run
 *   bin     : counts[i] (uint64 [nb], zeroed) += the rows with edges[i] <= z < edges[i+1] (edges double [nb + 1],
 *             non-decreasing; NaN and rows outside [edges[0], edges[nb]) are not counted); sums[i] (double [nb],
 *             zeroed) += their weights when w is not NULL.  inv_h > 0: the edges are evenly spaced about 1 / inv_h apart,
 *             and the bin is guessed from (z - edges[0]) inv_h and corrected against them; inv_h = 0: binary search.
 *             nb <= nbk_zh_smem_bins() accumulates in per-CTA shared memory, more bins in global atomics
 *   spline  : out[i] (double) = the cubic B-spline of knots t[nt] and coefficients c (nt - 4 used) at z[i], as FITPACK's
 *             splev with ext 0 (extrapolate), 1 (zeros), 2 (raise: the extrapolated value is written) or 3 (const);
 *             *outside (device uint64) += the rows outside [t[3], t[nt - 4]] */
int64_t nbk_zh_smem_bins(void);
int64_t nbk_zh_partials(void);
int nbk_zh_moments(const void *z, int dtype, int64_t n, double *partial, double *out, void *stream);
int nbk_zh_bin(const void *z, int dtype, const void *w, int wdtype, int64_t n, const double *edges, int64_t nb,
               double inv_h, uint64_t *counts, double *sums, void *stream);
int nbk_zh_spline(const void *z, int dtype, int64_t n, const double *t, int64_t nt, const double *c, int ext, double *out,
                  uint64_t *outside, void *stream);

/* HOD population (source/catalog/halos.py: HaloCatalog.populate; DESIGN.md 4.13).  n halos at global rows
 * h0 .. h0 + n - 1; every uniform is a SplitMix64 hash of (seed, stream, global halo row, draw index).
 *   occupy : Zheng07.  counts[i] (int64 [2 n]) = N_cen of halo i (Bernoulli, stream 0 draw 0) and counts[n + i] = N_sat
 *            (exact Poisson, stream 0 draws 1 ..), with M0 = 10^logM0, M1 = 10^logM1 and the satellite mean times the
 *            central probability when modulate is non-zero; mass (float32 / float64) in Msun/h
 *   occupy_smhm : Leauthaud11, the same draws and counts.  The cubic spline (t [nt], c, device doubles, FITPACK splev,
 *            extrapolated) maps log10 M to the mean log10 M*; <N_cen> = erfc((threshold - log10 M*) / (sqrt 2 scatter)) / 2,
 *            <N_sat> = (M / Msat)^alphasat exp(-Mcut / M), times <N_cen> when modulate is non-zero.  Hearin15 when pct
 *            (double [n], the halo's percentile in its mass bin) is not NULL: both means get the Heaviside
 *            assembly-bias shift of strength Acen / Asat (in [-1, 1]) up for pct > split, down otherwise
 *   scan   : offsets (int64 [n2 + 1]) = 0 and the inclusive sum of the n2 counts; work: nbk_hod_scan_workspace(n2) bytes
 *   emit   : galaxy row r < ngal = offsets[2 n] belongs to entry e with offsets[e] <= r < offsets[e + 1]: the central of
 *            halo e (e < n) or satellite k = r - offsets[e] of halo e - n (stream 1, draws 8 k .. 8 k + 6).  hpos, hvel,
 *            pos, vel, voff are (n or ngal, 3) of dtype (NBK_F4 / NBK_F8); mass, radius (proper Mpc/h), conc are double.
 *            Positions wrap into [0, box_host[d]); voff = vel * rsd; hcd = distance from the halo centre; gnewton = G in
 *            (km/s)^2 Mpc / Msun; table (2 K doubles) holds ln I and d ln I / ds of the Jeans integral at s0 + k hs */
int64_t nbk_hod_scan_workspace(int64_t n2);
int nbk_hod_occupy(const void *mass, int mdtype, int64_t n, int64_t h0, double logMmin, double sigma_logM, double M0,
                   double M1, double alpha, int modulate, uint64_t seed, int64_t *counts, void *stream);
int nbk_hod_occupy_smhm(const void *mass, int mdtype, int64_t n, int64_t h0, const double *t, int64_t nt, const double *c,
                        double threshold, double scatter, double Msat, double Mcut, double alphasat, int modulate,
                        const double *pct, double split, double Acen, double Asat, uint64_t seed, int64_t *counts,
                        void *stream);
int nbk_hod_scan(const int64_t *counts, int64_t n2, int64_t *offsets, void *work, int64_t work_bytes, void *stream);
int nbk_hod_emit(const int64_t *offsets, int64_t n, int64_t ngal, int64_t h0, const void *hpos, const void *hvel, int dtype,
                 const double *mass, const double *radius, const double *conc, const double *box_host, double gnewton,
                 double rsd, const double *table, int64_t K, double s0, double hs, uint64_t seed, void *pos, void *vel,
                 void *voff, double *hcd, int32_t *gal_type, int64_t *halo_id, void *stream);

/* elementwise helpers behind RealField/ComplexField `[...] = v`, `*= a`, `+= other`
 * (source/mesh/catalog.py:203,354,396-398; fftpower.py:128).  n counts REAL scalars. */
int nbk_fill(void *x, int dtype, int64_t n, double value, void *stream);
int nbk_scale(void *x, int dtype, int64_t n, double a, void *stream);
int nbk_axpy(void *y, const void *x, int dtype, int64_t n, double a, void *stream);
/* csum (source/mesh/catalog.py:388): out1 device double[1], accumulated into */
int nbk_sum(const void *x, int dtype, int64_t n, double *out1, void *stream);

#ifdef __cplusplus
}
#endif
#endif
