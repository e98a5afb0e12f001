"""
TEST INFRASTRUCTURE -- helpers of tests/test_gpu_mesh_layouts.py and tests/test_gpu_slab_route.py (never imported by
the product):

  * the slab layouts the Fourier- and real-space kernels take, as P virtual ranks of one array: the transposed y slabs
    [y_n][Nx][Nzc] that the slab FFT leaves on every GPU when P > 1, and the real x slabs [x_n][Ny][Nz];
  * float64 references on full (uncompressed) meshes where pmesh_oracle only knows the Hermitian half;
  * particle positions on and around the cell boundaries of the paint index arithmetic, and the CPU checks that show
    the positions do land there;
  * the particle routing between x slabs: positions around the slab edges and the route's float32 rejection edges, and
    the ranks a paint / readout stencil touches;
  * the fixed-point contract of the tiled paint: the scale the kernel derives from the masses, the exact NNB result it
    implies, and a per-cell error bound for the other windows.
"""
import numpy as np

from . import pmesh_oracle as po

# leftmost-cell offsets of the windows, i0 = floor(g + A) + B (csrc/paint.cu WinOff)
WIN_A = {"nnb": 0.5, "cic": 0.0, "tsc": 0.5, "pcs": 0.0}
WIN_B = {"nnb": 0, "cic": 0, "tsc": -1, "pcs": -1}
# largest |dW/dd| of the 1-D window weights (TSC: 2x at x = 1/2; PCS: (12x - 9x^2)/6 at x = 2/3)
WIN_SLOPE = {"nnb": 0.0, "cic": 1.0, "tsc": 1.0, "pcs": 2.0 / 3.0}


# ----------------------------------------------------------------------------------------------
# slab layouts
# ----------------------------------------------------------------------------------------------
def rank_counts(n, choices=(2, 3, 4)):
    """the virtual rank counts P in `choices` that divide the axis length n"""
    return [p for p in choices if n % p == 0]


def split_transposed(c, P):
    """rank r of P: y rows [r y_n, (r+1) y_n) of every x, stored transposed [y_n][Nx][Nzc] as its own array"""
    y_n = c.shape[1] // P
    return [np.ascontiguousarray(c[:, r * y_n:(r + 1) * y_n, :].transpose(1, 0, 2)) for r in range(P)]


def join_transposed(parts):
    """inverse of split_transposed"""
    return np.concatenate([np.asarray(p).transpose(1, 0, 2) for p in parts], axis=1)


def split_x(a, P):
    """rank r of P: x planes [r x_n, (r+1) x_n) as its own array"""
    x_n = a.shape[0] // P
    return [np.ascontiguousarray(a[r * x_n:(r + 1) * x_n]) for r in range(P)]


# ----------------------------------------------------------------------------------------------
# spectra and coordinates
# ----------------------------------------------------------------------------------------------
def spectra(N, rng, dtype="f8"):
    """(compressed, full) spectrum of a random real field: rfftn and fftn / prod(N), the full one being the Hermitian
    completion of the compressed one"""
    r = rng.standard_normal(tuple(N))
    c, f = np.fft.rfftn(r) / r.size, np.fft.fftn(r) / r.size
    cd = "c8" if dtype == "f4" else "c16"
    return c.astype(cd), f.astype(cd)


def k_coords(N, L, coord_dtype="f8", kind="wavenumber", fullz=False):
    """po.k_coords with the option of all Nz labels along z (the NBK_LAYOUT_FULLZ layout)"""
    if not fullz:
        return po.k_coords(N, L, coord_dtype, kind)
    L = np.asarray(L, dtype="f8") * np.ones(3)
    ct = np.dtype(coord_dtype).type
    out = []
    for d in range(3):
        j = po.freq_index(int(N[d]))
        unit = (2 * np.pi / L[d]) if kind == "wavenumber" else (2 * np.pi / N[d])
        shape = [1, 1, 1]
        shape[d] = len(j)
        out.append((j.astype(ct) * ct(unit)).reshape(shape))
    return out


def interlace_ref(c1, c2, N, L, fullz=False):
    """0.5 c1 + 0.5 c2 exp(0.5j sum_i k_i H_i) in f8 -- po.interlace_combine on either z layout"""
    H = np.asarray(L, dtype="f8") / np.asarray(N)
    k = k_coords(N, L, "f8", fullz=fullz)
    kH = sum(k[i] * H[i] for i in range(3))
    return c1 * 0.5 + c2 * 0.5 * np.exp(0.5j * kH)


def recon_ref(delta_k, N, L, axis, R, bias, f, los, fullz=False):
    """recon_oracle.displacement_modes on either z layout"""
    k = k_coords(N, L, "f8", fullz=fullz)
    k2 = sum(ki ** 2 for ki in k)
    k2 = np.where(k2 == 0, 1.0, k2)
    mu = sum(k[i] * los[i] for i in range(3)) / k2 ** 0.5
    v = delta_k * np.exp(-0.5 * k2 * R ** 2)
    v = v / (bias * (1 + f / bias * mu ** 2))
    return 1j * k[axis] / k2 * v


def mirror_dirs(N, L):
    """(direction of k, direction the unstored mirror mode -k carries on a full mesh) on the compressed layout, f8:
    every component flips sign except at the Nyquist index, whose label stays -N/2 (khat := 0 at k = 0)"""
    k = k_coords(N, L, "f8")
    m = []
    for d in range(3):
        j = po.freq_index(int(N[d]), compressed=(d == 2))
        keep = (2 * j == -int(N[d])).reshape(k[d].shape)
        m.append(np.where(keep, k[d], -k[d]))
    kn = np.sqrt(sum(x ** 2 for x in k))
    inv = np.where(kn == 0, 0.0, 1.0 / np.where(kn == 0, 1.0, kn))
    return [x * inv for x in k], [x * inv for x in m]


def project_sums_anti(y3d, x3d, edges, los, poles):
    """project_sums of a statistic with y(-k) = -conj y(k) (hermitian = 2): i y is Hermitian, and multiplying by i is
    exact, so the sums are -i times the Hermitian sums of i y"""
    xs, ms, ys, ns = po.project_sums(1j * y3d, x3d, edges, los, poles)
    return xs, ms, -1j * ys, ns


# ----------------------------------------------------------------------------------------------
# positions at the cell boundaries of the paint index arithmetic
# ----------------------------------------------------------------------------------------------
def _ulp_neighbours(v, dtype, k=3):
    v = np.asarray(v, dtype=dtype)
    out = [v]
    up, dn = v, v
    for _ in range(k):
        up = np.nextafter(up, np.asarray(np.inf, dtype=dtype))
        dn = np.nextafter(dn, np.asarray(-np.inf, dtype=dtype))
        out += [up, dn]
    return out


def boundary_values(N, L, dtype):
    """per axis: the coordinate values the generator targets -- the boundaries of cells k in {0, 1, N/2, N-1, N} for
    both window offsets (g and g + 1/2 integer), |g| just below / above 2^22 on both sides of zero, |x| ~ 1e3 L, exactly
    L, and -0.0 -- each with its +-1..3 ulp neighbours in `dtype`"""
    out = []
    for d in range(3):
        n, l = int(N[d]), float(L[d])
        vals = []
        for k in (0, 1, n // 2, n - 1, n):
            for half in (0.0, 0.5):
                vals += _ulp_neighbours((k - half) * l / n, dtype)
        for s in (1.0, -1.0):
            vals += _ulp_neighbours(s * 4194304.0 * l / n, dtype)
            vals += _ulp_neighbours(s * 1e3 * l + 0.37 * l / n, dtype)
        vals += _ulp_neighbours(l, dtype)
        # the ulp neighbours of 0 are denormals, which x * N/L may flush to zero: the smallest normal numbers as well
        for s in (1.0, -1.0):
            vals += _ulp_neighbours(s * np.finfo(dtype).tiny, dtype, 1)
        # (unique() merges -0.0 into 0.0: appended after it)
        out.append(np.append(np.unique(np.asarray(vals, dtype=dtype)), np.asarray(-0.0, dtype=dtype)))
    return out


def boundary_positions(N, L, dtype, n_total=100000, repeat=8, seed=0):
    """positions whose coordinate along one axis is a boundary value (the other two uniform in the box), `repeat`
    times each, padded with uniform particles to n_total.  Returns (pos, number of boundary rows); boundary rows first."""
    rng = np.random.RandomState(seed)
    L = np.asarray(L, dtype="f8")
    rows = []
    for d, vals in enumerate(boundary_values(N, L, dtype)):
        v = np.repeat(vals, repeat)
        p = rng.uniform(0, 1, size=(len(v), 3)) * L
        p = p.astype(dtype)
        p[:, d] = v
        rows.append(p)
    special = np.concatenate(rows)
    pad = (rng.uniform(0, 1, size=(max(0, n_total - len(special)), 3)) * L).astype(dtype)
    return np.concatenate([special, pad]), len(special)


def exact_cell(x, n, l, resampler):
    """unwrapped leftmost cell along one axis in the exact f8 arithmetic of the contract: floor(fl(x * fl(N/L)) + A) + B"""
    g = np.asarray(x).astype("f8") * (float(n) / float(l))
    return np.floor(g + WIN_A[resampler]).astype("i8") + WIN_B[resampler]


def fast_tile_needs_f8(x, n, l, resampler):
    """True where the float32 tile id of csrc/paint.cu (tile_fast, N/L not a power of two) is not decisive and the
    count pass recomputes it in f8: |frac(g32 + A) - 1/2| >= lim, lim = 1/2 - (3e-7 (n + 2) + 1e-6), all in float32"""
    f4 = np.float32
    g = np.asarray(x, dtype=f4) * f4(float(n) / float(l))
    if WIN_A[resampler]:
        g = g + f4(WIN_A[resampler])
    fr = (g - np.floor(g)).astype(f4)
    lim = f4(0.5) - (f4(3e-7) * f4(n + 2) + f4(1e-6))
    return ~(np.abs(fr - f4(0.5)) < lim)


# ----------------------------------------------------------------------------------------------
# particle routing between x slabs (csrc/route.cu)
# ----------------------------------------------------------------------------------------------
def route_margin(Nx):
    """the float32 margin of the route's rejection test, in cells: 1e-3 + 4e-7 Nx, in float32 as a multiply then an add
    (csrc/route.cu is compiled with --fmad=false, so the device does not contract them into an FMA either; the +-3
    float32 ulp neighbours of slab_edge_values would straddle an edge one ulp away as well)"""
    f4 = np.float32
    return f4(1e-3) + f4(4e-7) * f4(Nx)


def route_reject_edges(Nx, P, s):
    """float32 grid coordinates (in_lo, in_hi) of every rank: a particle with in_lo < fl32(x) fl32(N/L) < in_hi is
    rejected in float32 (never examined in f8)"""
    f4 = np.float32
    x_n, m = Nx // P, route_margin(Nx)
    return [(f4(r * x_n) + f4(s) + m, f4((r + 1) * x_n) - f4(s) - m) for r in range(P)]


def slab_edge_targets(Nx, P, smoothings):
    """the grid coordinates b + d the slab-edge generator targets: every slab boundary b = r x_n (r = 0 .. P, the seam
    at 0 = Nx included) with d in {-s-1, -s, -1/2, 0, 1/2, s, s+1} for every smoothing s"""
    x_n = Nx // P
    t = set()
    for r in range(P + 1):
        for s in smoothings:
            for d in (-s - 1, -s, -0.5, 0.0, 0.5, s, s + 1):
                t.add(float(r * x_n + d))
    return sorted(t)


def slab_edge_values(Nx, L, P, smoothings, dtype, k=3):
    """x coordinates (in `dtype`) around the slab edges of the routing: every target of slab_edge_targets and every
    float32 rejection edge of route_reject_edges, each with its +-0..k ulp neighbours (float32 ulps for the rejection
    edges, which live in float32); the seam targets moved 1 .. 3 box lengths out on both sides; +0 and -0"""
    L = float(L)
    sc32 = np.float32(float(Nx) / L)
    vals = []
    targets = slab_edge_targets(Nx, P, smoothings)
    for g in targets:
        vals += _ulp_neighbours(g * L / Nx, dtype, k)
    for s in smoothings:
        for lo, hi in route_reject_edges(Nx, P, s):
            for e in (lo, hi):
                # the float32 x whose fl32(x * fl32(N/L)) is nearest to the edge, and its float32 neighbours
                x = np.float32(np.float64(e) / np.float64(sc32))
                vals += [np.asarray(v, dtype=dtype) for v in _ulp_neighbours(x, np.float32, k)]
    seam = [g for g in targets if abs(g) <= max(smoothings) + 1]
    for j in (-3, -2, -1, 1, 2, 3):
        for g in seam:
            vals += _ulp_neighbours((g + j * Nx) * L / Nx, dtype, 1)
    out = np.unique(np.asarray(vals, dtype=dtype))
    return np.append(out, np.asarray([0.0, -0.0], dtype=dtype))


def slab_edge_positions(N, L, P, smoothings, dtype, n_uniform=5000, seed=0):
    """positions whose x is a slab_edge_values value (y, z uniform in the box) followed by n_uniform uniform
    particles.  Returns (pos, number of edge rows)"""
    rng = np.random.RandomState(seed)
    L = np.asarray(L, dtype="f8")
    v = slab_edge_values(int(N[0]), L[0], P, smoothings, dtype)
    edge = (rng.uniform(0, 1, size=(len(v), 3)) * L).astype(dtype)
    edge[:, 0] = v
    uni = (rng.uniform(0, 1, size=(n_uniform, 3)) * L).astype(dtype)
    return np.concatenate([edge, uni]), len(v)


def stencil_ranks(pos, N, L, P, resampler, shifts):
    """bitmask (int64) of the ranks of P x slabs that own a plane the window stencil of each particle touches, at any
    of `shifts` -- from the exact paint / readout cell arithmetic (po.grid_coords, po.window_1d), not from the route"""
    Nx = int(N[0])
    x_n = Nx // P
    sup = po.SUPPORT[resampler]
    mask = np.zeros(len(pos), dtype="i8")
    for shift in shifts:
        g = po.grid_coords(pos, N, L, shift)[:, 0]
        i0 = po.window_1d(g, resampler)[0]
        for j in range(sup):
            mask |= np.left_shift(1, ((i0 + j) % Nx) // x_n).astype("i8")
    return mask


# ----------------------------------------------------------------------------------------------
# fixed-point contract of the tiled paint
# ----------------------------------------------------------------------------------------------
def fixed_point_scale(mass):
    """M of the tiled paint: the power of two above fl32(fl32(max |mass|) * 1.0000001f) (1 without masses / all zero)"""
    if mass is None:
        return 1.0
    a = np.abs(np.asarray(mass)).astype(np.float32)
    mx = (a * np.float32(1.0000001)).max() if len(a) else np.float32(0)
    if not mx > 0:
        return 1.0
    _, e = np.frexp(np.float64(mx))
    return float(2.0 ** int(e))


def nnb_fixed_point(pos, mass, N, L, shift=0.0):
    """what the tiled paint must give for NNB, bit for bit: every deposit is round-half-even(m 2^31 / M), the cell is
    the exact integer sum times M / 2^31 (f8)"""
    N = np.asarray(N, dtype="i8")
    M = fixed_point_scale(mass)
    m = np.ones(len(pos)) if mass is None else np.asarray(mass, dtype="f8")
    q = np.rint(m * (2.0 ** 31 / M)).astype("i8")
    c = po.cell_index(pos, N, L, "nnb", shift)
    flat = (c[:, 0] * N[1] + c[:, 1]) * N[2] + c[:, 2]
    acc = np.zeros(int(np.prod(N)), dtype="i8")
    np.add.at(acc, flat, q)
    return (acc.astype("f8") * (M / 2.0 ** 31)).reshape(tuple(N))


def deposit_bound(pos, mass, N, L, resampler, shift=0.0):
    """per-cell bound on |tiled - exact| (f8 mesh): sum over the deposits into the cell of M 2^-32 (rounding of the
    fixed-point deposit) + |m| 3 c 2^-28 (the 28-bit truncated fraction of the record moves each of the three 1-D weights
    by < c 2^-28, c = largest weight slope; NNB: 0), plus a few f8 roundings of the value"""
    N = np.asarray(N, dtype="i8")
    M = fixed_point_scale(mass)
    am = np.ones(len(pos)) if mass is None else np.abs(np.asarray(mass, dtype="f8"))
    g = po.grid_coords(pos, N, L, shift)
    i0 = [po.window_1d(g[:, d], resampler)[0] for d in range(3)]
    sup = po.SUPPORT[resampler]
    cnt = np.zeros(int(np.prod(N)))
    msum = np.zeros(int(np.prod(N)))
    for rx in range(sup):
        for ry in range(sup):
            for rz in range(sup):
                flat = (((i0[0] + rx) % N[0]) * N[1] + (i0[1] + ry) % N[1]) * N[2] + (i0[2] + rz) % N[2]
                cnt += np.bincount(flat, minlength=cnt.size)
                msum += np.bincount(flat, weights=am, minlength=cnt.size)
    bound = cnt * (M * 2.0 ** -32) * (1 + 1e-6) + msum * (3 * WIN_SLOPE[resampler] * 2.0 ** -28 + 1e-15)
    return bound.reshape(tuple(N)), cnt.reshape(tuple(N))
