"""
TEST INFRASTRUCTURE -- CPU oracle for the FFTPower hot path.  NOT product code:
only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import it.  The product path (nbodykit_b200) never does.

It restates, in NumPy, the arithmetic of the un-vendored dependency `pmesh`
(github rainwoodman/pmesh, unpinned in /root/reference/requirements.txt:7; last
compatibility note "pmesh 0.1.56", CHANGES.rst:11) as used at the reference's own
call sites, plus NumPy restatements of the reference's pure-NumPy steps
(project_to_basis, Compensate*, MPIRandomState) so the oracle can travel to the GPU
box where /root/reference does not exist.

PARITY STATUS
  * project_to_basis, Compensate*, MPIRandomState restatements are PINNED: they are
    checked against the reference's own code (loaded verbatim by oracle/refload.py)
    in tests/test_oracle_vs_reference.py and through golden vectors generated from
    the reference code (tests/golden/make_golden.py).
  * shell indexing is PINNED by the reference fixture nbodykit/tests/data/dataset_2d.json
    (k-marginal mode counts, tests/golden/dataset_2d_modes.json) -- reproduced only
    with float32 coordinate arithmetic, which is therefore the contract.
  * the pmesh pieces (window paint, r2c normalisation, interlacing) are "parity
    unpinned" per cell/mode: the reference's tests hold no literal mesh or delta(k)
    values.  They are pinned only through the reference's own statistical assertions
    (tests/test_reference_assertions.py: chi^2 < 1 for CIC/TSC compensated shot noise,
    the interlacing sign test, N1=96 doc known answer).

Semantics follow SURVEY.md Appendix B.
"""
import numpy as np

# ----------------------------------------------------------------------------------------------
# windows  (pmesh.window.methods[...].support used at source/mesh/catalog.py:194,271-273)
# ----------------------------------------------------------------------------------------------
SUPPORT = {"nnb": 1, "nearest": 1, "cic": 2, "tsc": 3, "pcs": 4}


def _tsc_kernel(x):
    x = np.abs(x)
    return np.where(x <= 0.5, 0.75 - x * x, np.where(x < 1.5, 0.5 * (1.5 - x) ** 2, 0.0))


def _pcs_kernel(x):
    x = np.abs(x)
    return np.where(x < 1.0, (4.0 - 6.0 * x * x + 3.0 * x ** 3) / 6.0,
                    np.where(x < 2.0, (2.0 - x) ** 3 / 6.0, 0.0))


def window_1d(g, resampler):
    """leftmost cell i0 (int64, un-wrapped) and the `support` 1-D weights for grid coordinates g (f8).

    CIC: i0 = floor(g), w = (1-d, d);  TSC: i0 = floor(g+0.5)-1, w_r = K(g-i0-r)  (SURVEY B.1, A6)
    """
    sup = SUPPORT[resampler]
    if resampler in ("nnb", "nearest"):
        i0 = np.floor(g + 0.5).astype(np.int64)
        return i0, [np.ones_like(g)]
    if resampler == "cic":
        i0f = np.floor(g)
        d = g - i0f
        return i0f.astype(np.int64), [1.0 - d, d]
    if resampler == "tsc":
        i0f = np.floor(g + 0.5) - 1.0
        d = g - i0f
        return i0f.astype(np.int64), [_tsc_kernel(d - r) for r in range(sup)]
    if resampler == "pcs":
        i0f = np.floor(g) - 1.0
        d = g - i0f
        return i0f.astype(np.int64), [_pcs_kernel(d - r) for r in range(sup)]
    raise ValueError("unknown resampler %s" % resampler)


def grid_coords(pos, Nmesh, BoxSize, shift=0.0, x_start=0):
    """g_d = fl(fl(double(pos_d) * fl(N_d/L_d)) + t_d), t = -x_start + shift   (SURVEY B.1)"""
    Nmesh = np.asarray(Nmesh, dtype="f8") * np.ones(3)
    BoxSize = np.asarray(BoxSize, dtype="f8") * np.ones(3)
    scale = Nmesh / BoxSize
    g = np.asarray(pos).astype("f8") * scale
    t = np.array([-float(x_start) + shift, shift, shift])
    return g + t


def paint(pos, mass, Nmesh, BoxSize, resampler="cic", shift=0.0, out=None, dtype="f8",
          x_start=0, x_n=None):
    """pm.paint(pos, mass=, resampler=, transform=affine[.shift(shift)], hold=True, out=)
    as called from source/mesh/catalog.py:287,295-296.  Periodic wrap in grid units; with a slab
    (x_start, x_n) stencil points falling outside the slab are dropped (pmesh ghost semantics, A8).
    Sums are formed in f8 and cast to `dtype` on return (the reference adds in mesh dtype; order of
    summation is unspecified there)."""
    N = (np.asarray(Nmesh, dtype="i8") * np.ones(3, dtype="i8"))
    if x_n is None:
        x_n = int(N[0])
    pos = np.asarray(pos)
    n = len(pos)
    if mass is None:
        mass = np.ones(n)
    mass = np.broadcast_to(np.asarray(mass, dtype="f8"), (n,))
    acc = np.zeros(x_n * int(N[1]) * int(N[2]), dtype="f8")
    if n:
        g = grid_coords(pos, N, BoxSize, shift, 0)
        i0 = []
        w = []
        for d in range(3):
            a, b = window_1d(g[:, d], resampler)
            i0.append(a)
            w.append(b)
        sup = SUPPORT[resampler]
        for rx in range(sup):
            ix = (i0[0] + rx) % N[0] - x_start
            okx = (ix >= 0) & (ix < x_n)
            for ry in range(sup):
                iy = (i0[1] + ry) % N[1]
                wxy = w[0][rx] * w[1][ry]
                for rz in range(sup):
                    iz = (i0[2] + rz) % N[2]
                    wt = wxy * w[2][rz] * mass
                    flat = (ix * N[1] + iy) * N[2] + iz
                    acc += np.bincount(flat[okx], weights=wt[okx], minlength=acc.size)
    acc = acc.reshape(x_n, int(N[1]), int(N[2]))
    if out is not None:
        out += acc.astype(out.dtype)
        return out
    return acc.astype(dtype)


def cell_index(pos, Nmesh, BoxSize, resampler="cic", shift=0.0):
    """wrapped leftmost-cell index (n,3) int64 -- the bit-exact part of the paint contract"""
    N = (np.asarray(Nmesh, dtype="i8") * np.ones(3, dtype="i8"))
    g = grid_coords(pos, N, BoxSize, shift, 0)
    return np.stack([window_1d(g[:, d], resampler)[0] % N[d] for d in range(3)], axis=1)


# ----------------------------------------------------------------------------------------------
# FFT  (RealField.r2c / ComplexField.c2r : forward normalised by 1/prod(N), backward unnormalised;
#       source/mesh/array.py:36-37, fftpower.py:126-128; SURVEY B.4)
# ----------------------------------------------------------------------------------------------
def _workers():
    import os
    return max(1, (os.cpu_count() or 1))


def r2c(real):
    import scipy.fft
    c = scipy.fft.rfftn(real, workers=_workers())
    c *= 1.0 / real.size
    return c.astype(np.complex64 if real.dtype == np.float32 else np.complex128, copy=False)


def c2r(cplx, Nmesh):
    import scipy.fft
    N = tuple(int(x) for x in (np.asarray(Nmesh, dtype="i8") * np.ones(3, dtype="i8")))
    r = scipy.fft.irfftn(cplx, s=N, workers=_workers()) * float(np.prod(N))
    return r.astype(np.float32 if cplx.dtype == np.complex64 else np.float64, copy=False)


# ----------------------------------------------------------------------------------------------
# coordinate arrays  (pm.k / field.x for complex fields; SURVEY A3, A12, B.5)
# ----------------------------------------------------------------------------------------------
def freq_index(N, compressed=False):
    """integer frequency labels j -> j if j < N/2 else j-N (Nyquist negative, meshtools.py:150-153)"""
    n = (N // 2 + 1) if compressed else N
    j = np.arange(n, dtype="i8")
    j[j >= (N + 1) // 2] -= N
    return j


def k_coords(Nmesh, BoxSize, coord_dtype="f4", kind="wavenumber"):
    """three broadcastable arrays shaped (N0,1,1),(1,N1,1),(1,1,N2/2+1).
    f4 (fixture-faithful default): k_d = fl32(f32(j_d) * f32(2 pi / L_d));  circular: f32(j)*f32(2 pi/N)"""
    N = (np.asarray(Nmesh, dtype="i8") * np.ones(3, dtype="i8"))
    L = np.asarray(BoxSize, dtype="f8") * np.ones(3)
    ct = np.dtype(coord_dtype).type
    out = []
    for d in range(3):
        j = freq_index(int(N[d]), compressed=(d == 2))
        unit = (2 * np.pi / L[d]) if kind == "wavenumber" else (2 * np.pi / N[d])
        k = j.astype(ct) * ct(unit)
        shape = [1, 1, 1]
        shape[d] = len(k)
        out.append(k.reshape(shape))
    return out


# ----------------------------------------------------------------------------------------------
# compensation  (restates source/mesh/catalog.py:449-594; validated against the reference's functions)
# ----------------------------------------------------------------------------------------------
COMPENSATION = {  # (interlaced, resampler) -> name  (get_compensation, source/mesh/catalog.py:419-447)
    (True, "cic"): "CompensateCIC", (True, "tsc"): "CompensateTSC", (True, "pcs"): "CompensatePCS",
    (False, "cic"): "CompensateCICShotnoise", (False, "tsc"): "CompensateTSCShotnoise",
    (False, "pcs"): "CompensatePCSShotnoise"}


def compensate(name, w, v):
    """v / prod_i f(w_i); w = circular coordinate arrays.  Same operation order and dtypes as the
    reference (factors are formed in w's dtype, divided into v one axis at a time)."""
    for i in range(3):
        wi = w[i]
        if name in ("CompensateCIC", "CompensateTSC", "CompensatePCS"):
            p = {"CompensateCIC": 2, "CompensateTSC": 3, "CompensatePCS": 4}[name]
            tmp = (np.sinc(0.5 * wi / np.pi)) ** p
            tmp[wi == 0.] = 1.
            v = v / tmp
        elif name == "CompensateCICShotnoise":
            v = v / (1 - 2. / 3 * np.sin(0.5 * wi) ** 2) ** 0.5
        elif name == "CompensateTSCShotnoise":
            s = np.sin(0.5 * wi) ** 2
            v = v / (1 - s + 2. / 15 * s ** 2) ** 0.5
        elif name == "CompensatePCSShotnoise":
            s = np.sin(0.5 * wi) ** 2
            v = v / (1 - 4. / 3. * s + 2. / 5. * s ** 2 - 4. / 315. * s ** 3) ** 0.5
        else:
            raise ValueError("compensation %s is not defined" % name)
    return v


def interlace_combine(c1, c2, Nmesh, BoxSize, coord_dtype="f4"):
    """c = 0.5 c1 + 0.5 c2 exp(0.5j sum_i k_i H_i)   (source/mesh/catalog.py:345-347)"""
    N = (np.asarray(Nmesh, dtype="i8") * np.ones(3, dtype="i8"))
    L = np.asarray(BoxSize, dtype="f8") * np.ones(3)
    H = L / N
    k = k_coords(N, L, coord_dtype)
    kH = sum(k[i] * H[i] for i in range(3))
    return (c1 * 0.5 + c2 * 0.5 * np.exp(0.5 * 1j * kH)).astype(c1.dtype)


# ----------------------------------------------------------------------------------------------
# project_to_basis  (restates algorithms/fftpower.py:507-701 + meshtools.py:104-215, vectorised over
# the whole field instead of per x-slab; per-element arithmetic and dtypes are identical)
# ----------------------------------------------------------------------------------------------
def _legendre_coeffs(ell):
    from scipy.special import legendre
    return np.asarray(legendre(ell).coeffs, dtype="f8")


def _legendre_horner(ell, mu):
    """numpy.poly1d.__call__ of scipy.special.legendre(ell) = polyval: Horner with f8 coefficients on mu.  The
    reference calls legendre(ell)(mu), which scipy 1.18's orthopoly1d routes to eval_legendre; a plain poly1d takes
    this Horner form, whose cancellation error grows past 1e-10 at ell = 16 and past 1 at ell = 40"""
    leg = np.zeros_like(mu, dtype="f8")
    for pv in _legendre_coeffs(ell):
        leg = leg * mu + pv
    return leg


def project_sums(y3d, x3d, edges, los=(0, 0, 1), poles=(), hermitian_symmetric=True, planes=None, legendre=None):
    """the raw per-bin sums of `project_to_basis` over the x-planes `planes` (default: all) -- what one MPI rank
    of the reference accumulates before the allreduce (fftpower.py:605-672).  Returns (xsum, musum, ysum, Nsum)
    shaped (Nx+2, Nmu+2) [ysum: (Nell, Nx+2, Nmu+2)].
    `legendre(ell, mu)` gives the weights (default: Horner on the coefficients of scipy.special.legendre, see
    _legendre_horner; pass scipy.special.eval_legendre above ell ~ 8, where the Horner form loses digits)."""
    legendre = _legendre_horner if legendre is None else legendre
    xedges, muedges = edges
    x2edges = np.asarray(xedges) ** 2
    Nx = len(xedges) - 1
    Nmu = len(muedges) - 1
    poles = list(poles)
    _poles = [0] + sorted(poles) if 0 not in poles else sorted(poles)
    if any(ell < 0 for ell in _poles):
        raise ValueError("in `project_to_basis`, multipole numbers must be non-negative integers")
    Nell = len(_poles)

    nbins = (Nx + 2) * (Nmu + 2)
    musum = np.zeros(nbins)
    xsum = np.zeros(nbins)
    ysum = np.zeros((Nell, nbins), dtype=np.complex128)
    Nsum = np.zeros(nbins, dtype="i8")

    # loop over x-planes to bound memory (the reference does the same, fftpower.py:605)
    x0, x1, x2 = x3d
    for islab in (range(y3d.shape[0]) if planes is None else planes):
        c0 = x0[islab].reshape(1, 1)
        c1 = x1[0]
        c2 = x2[0]
        # norm2 = sum(coords(i)**2): ((0 + x0^2) + x1^2) + x2^2  (meshtools.py:117)
        xslab = (0 + c0 ** 2) + c1 ** 2 + c2 ** 2
        dig_x = np.digitize(xslab.flat, x2edges)
        xslab = xslab ** 0.5
        with np.errstate(invalid="ignore", divide="ignore"):
            mu = (0 + c0 * los[0] + c1 * los[1] + c2 * los[2]) / xslab
        mu[xslab == 0.0] = 0.0
        dig_mu = np.digitize(mu.flat, muedges)
        multi_index = dig_x * (Nmu + 2) + dig_mu

        if hermitian_symmetric:
            nonsing = np.broadcast_to(c2 > 0., xslab.shape)
            hw = np.ones(xslab.shape, dtype="f4")
            hw[nonsing] = 2.
        else:
            nonsing = None
            hw = 1.

        xsum += np.bincount(multi_index, weights=(xslab * hw).flat, minlength=nbins)
        Nsum += np.bincount(multi_index, weights=(np.ones_like(xslab) * hw).flat,
                            minlength=nbins).astype("i8")
        yplane = y3d[islab]
        for iell, ell in enumerate(_poles):
            # (a float32 mu widens exactly, as the kernel widens it)
            leg = np.asarray(legendre(ell, mu.astype("f8")), dtype="f8")
            wy = (leg * yplane).astype(np.complex128)
            if hermitian_symmetric:
                if ell % 2:
                    wy.real[nonsing] = 0.
                    wy.imag[nonsing] *= 2.
                else:
                    wy.real[nonsing] *= 2.
                    wy.imag[nonsing] = 0.
            wy *= (2. * ell + 1.)
            ysum[iell] += np.bincount(multi_index, weights=wy.real.flat, minlength=nbins)
            ysum[iell] += 1j * np.bincount(multi_index, weights=wy.imag.flat, minlength=nbins)
        musum += np.bincount(multi_index, weights=(mu * hw).flat, minlength=nbins)

    musum = musum.reshape(Nx + 2, Nmu + 2)
    xsum = xsum.reshape(Nx + 2, Nmu + 2)
    Nsum = Nsum.reshape(Nx + 2, Nmu + 2)
    ysum = ysum.reshape(Nell, Nx + 2, Nmu + 2)
    return xsum, musum, ysum, Nsum


def project_to_basis(y3d, x3d, edges, los=(0, 0, 1), poles=(), hermitian_symmetric=True, legendre=None):
    """y3d: ndarray (N0,N1,N2c); x3d: 3 broadcastable coordinate arrays (their dtype is part of the
    contract).  Returns exactly what the reference returns:
    (xmean_2d, mumean_2d, y2d, N_2d), (xmean_1d, poles, N_1d) | None
    (`legendre`: see project_sums)"""
    poles = list(poles)
    _poles = [0] + sorted(poles) if 0 not in poles else sorted(poles)
    if any(ell < 0 for ell in _poles):
        raise ValueError("in `project_to_basis`, multipole numbers must be non-negative integers")
    ell_idx = [_poles.index(l) for l in poles]
    xsum, musum, ysum, Nsum = project_sums(y3d, x3d, edges, los, poles, hermitian_symmetric, legendre=legendre)
    return finish_projection(xsum, musum, ysum, Nsum, len(poles) > 0, ell_idx)


def finish_projection(xsum, musum, ysum, Nsum, do_poles, ell_idx):
    """fold the mu==1 overflow bin and form means  (fftpower.py:674-701)"""
    ysum = ysum.copy(); musum = musum.copy(); xsum = xsum.copy(); Nsum = Nsum.copy()
    ysum[..., -2] += ysum[..., -1]
    musum[:, -2] += musum[:, -1]
    xsum[:, -2] += xsum[:, -1]
    Nsum[:, -2] += Nsum[:, -1]
    sl = slice(1, -1)
    with np.errstate(invalid="ignore", divide="ignore"):
        y2d = (ysum[0, ...] / Nsum)[sl, sl]
        xmean_2d = (xsum / Nsum)[sl, sl]
        mumean_2d = (musum / Nsum)[sl, sl]
        N_2d = Nsum[sl, sl]
        pole_result = None
        if do_poles:
            N_1d = Nsum[sl, sl].sum(axis=-1)
            xmean_1d = xsum[sl, sl].sum(axis=-1) / N_1d
            poles = ysum[:, sl, sl].sum(axis=-1) / N_1d
            poles = poles[ell_idx, ...]
            pole_result = (xmean_1d, poles, N_1d)
    return (xmean_2d, mumean_2d, y2d, N_2d), pole_result


# ----------------------------------------------------------------------------------------------
# MPIRandomState / UniformCatalog  (restates mpirng.py:135-251, uniform.py:85-101 for one rank)
# ----------------------------------------------------------------------------------------------
class SerialMPIRandomState(object):
    def __init__(self, seed, size, chunksize=100000):
        self.size = size
        self.chunksize = chunksize
        self.nchunks = (size + chunksize - 1) // chunksize
        self._serial_rng = np.random.RandomState(seed)

    def _call(self, sampler, itemshape, dtype):
        # every call re-draws the seed table from the serial rng (mpirng.py:224)
        seeds = self._serial_rng.randint(0, high=0xffffffff, size=self.nchunks)
        r = np.zeros((self.size,) + tuple(itemshape), dtype=dtype)
        for ichunk in range(self.nchunks):
            lo = ichunk * self.chunksize
            nreq = min(self.size - lo, self.chunksize)
            rng = np.random.RandomState(seeds[ichunk])
            r[lo:lo + nreq] = sampler(rng, (nreq,) + tuple(itemshape))
        return r

    def uniform(self, low=0., high=1.0, itemshape=(), dtype="f8"):
        return self._call(lambda rng, size: rng.uniform(low=low, high=high, size=size), itemshape, dtype)

    def normal(self, loc=0, scale=1, itemshape=(), dtype="f8"):
        return self._call(lambda rng, size: rng.normal(loc=loc, scale=scale, size=size), itemshape, dtype)


def uniform_catalog(nbar, BoxSize, seed, dtype="f8"):
    """Position, Velocity of UniformCatalog(nbar, BoxSize, seed) on one rank (uniform.py:85-101)"""
    L = np.empty(3, dtype="f8")
    L[:] = BoxSize
    N = np.random.RandomState(seed).poisson(nbar * np.prod(L))
    rng = SerialMPIRandomState(seed, N)
    pos = (rng.uniform(itemshape=(3,)) * L).astype(dtype)
    vel = (rng.uniform(itemshape=(3,)) * L * 0.01).astype(dtype)
    return pos, vel


# ----------------------------------------------------------------------------------------------
# the whole FFTPower flow on the CPU  (fftpower.py:230-334 + catalog.py:155-403 + base/mesh.py:256-338)
# ----------------------------------------------------------------------------------------------
def paint_field(pos, Nmesh, BoxSize, resampler="cic", interlaced=False, weight=None, value=None,
                dtype="f8", coord_dtype="f4"):
    """CatalogMesh.to_real_field: returns (1+delta field, attrs)"""
    N = (np.asarray(Nmesh, dtype="i8") * np.ones(3, dtype="i8"))
    L = np.asarray(BoxSize, dtype="f8") * np.ones(3)
    n = len(pos)
    w = np.ones(n) if weight is None else np.asarray(weight, dtype="f8")
    v = np.ones(n) if value is None else np.asarray(value, dtype="f8")
    if not interlaced:
        real = paint(pos, w * v, N, L, resampler, 0.0, dtype=dtype)
    else:
        r1 = paint(pos, w * v, N, L, resampler, 0.0, dtype=dtype)
        r2 = paint(pos, w * v, N, L, resampler, 0.5, dtype=dtype)
        c = interlace_combine(r2c(r1), r2c(r2), N, L, coord_dtype)
        real = c2r(c, N)
    W = float(w.sum())
    W2 = float((w ** 2).sum())
    nbar = W / float(np.prod(N))
    attrs = dict(N=n, W=W, W2=W2, num_per_cell=nbar,
                 shotnoise=(float(np.prod(L)) * W2 / W ** 2) if W != 0 else np.nan)
    if nbar > 0:
        real = (real / real.dtype.type(nbar)).astype(real.dtype)
    else:
        real[...] = 1
    return real, attrs


def fftpower(pos, Nmesh, BoxSize, mode="1d", resampler="cic", interlaced=False, compensated=True,
             weight=None, value=None, dtype="f8", los=(0, 0, 1), Nmu=5, dk=None, kmin=0., kmax=None,
             poles=(), coord_dtype="f4"):
    """FFTPower(cat.to_mesh(...), mode=...) restated end to end; returns dict of arrays + attrs"""
    N = (np.asarray(Nmesh, dtype="i8") * np.ones(3, dtype="i8"))
    L = np.asarray(BoxSize, dtype="f8") * np.ones(3)
    real, attrs = paint_field(pos, N, L, resampler, interlaced, weight, value, dtype, coord_dtype)
    c = r2c(real)
    if compensated:
        wc = k_coords(N, L, coord_dtype, kind="circular")
        c = compensate(COMPENSATION[(interlaced, resampler)], wc, c).astype(c.dtype)
    return power_from_complex(c, None, N, L, mode, los, Nmu, dk, kmin, kmax, poles, coord_dtype, attrs)


def power_from_complex(c1, c2, Nmesh, BoxSize, mode="1d", los=(0, 0, 1), Nmu=5, dk=None, kmin=0.,
                       kmax=None, poles=(), coord_dtype="f4", attrs=None):
    N = (np.asarray(Nmesh, dtype="i8") * np.ones(3, dtype="i8"))
    L = np.asarray(BoxSize, dtype="f8") * np.ones(3)
    p3d = c1 * np.conj(c1 if c2 is None else c2)      # fftpower.py:115-117
    p3d[0, 0, 0] = 0                                  # :119-124
    p3d = p3d * p3d.dtype.type(L.prod())              # :128
    if mode == "1d":
        Nmu = 1
    if dk is None:
        dk = 2 * np.pi / L.min()
    if kmax is None:
        kmax = np.pi * N.min() / L.max() + dk / 2
    kedges = np.arange(kmin, kmax, dk)
    muedges = np.linspace(-1, 1, Nmu + 1, endpoint=True)
    x3d = k_coords(N, L, coord_dtype)
    res, pole_res = project_to_basis(p3d, x3d, [kedges, muedges], los=los, poles=poles)
    out = dict(kedges=kedges, muedges=muedges, k=res[0], mu=res[1], power=res[2], modes=res[3],
               attrs=dict(attrs or {}))
    if pole_res is not None:
        out.update(poles_k=pole_res[0], poles_power=pole_res[1], poles_modes=pole_res[2])
    return out
