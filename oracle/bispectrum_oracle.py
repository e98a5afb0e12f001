"""
TEST INFRASTRUCTURE -- float64 NumPy oracle for FFTBispectrum (nbodykit_b200/algorithms/bispectrum.py, DESIGN.md 4.14).
NOT product code.

Input: the Hermitian-compressed spectrum `half` (Nx, Ny, Nz//2+1) of a real field, normalised as compute(mode='complex')
(delta(q), forward transform / N^3).  Shells follow FFTPower's k bins at float32 coordinates (pmesh_oracle.k_coords and
numpy.digitize of |k|^2 against kedges^2); the k = 0 mode is in no shell.  Two independent forms:

  fft_form    -- the estimator's contract: I_i = c2r(c 1_Si), J_i = c2r(1_Si) (unnormalised backward transforms, numpy
                 irfftn * N^3), S_ijl = sum_x I_i I_j I_l, T_ijl = sum_x J_i J_j J_l / N^3, B = V^2 S / sum_x J J J
  direct_form -- no FFT: sum over q1 in S_i, q2 in S_j with q3 = -(q1 + q2) modulo the grid in S_l of
                 c(q1) c(q2) c(q3); T counts those ordered triplets.  O(|S_i| |S_j|) per shell pair: up to ~16^3.
"""
import numpy as np

from . import pmesh_oracle as po


def triples(kedges):
    """sorted shell triples i <= j <= l with kedges[l] < kedges[i+1] + kedges[j+1], lexicographic"""
    e = np.asarray(kedges, dtype="f8")
    n = len(e) - 1
    return np.array([(i, j, l) for i in range(n) for j in range(i, n) for l in range(j, n)
                     if e[l] < e[i + 1] + e[j + 1]], dtype="i8").reshape(-1, 3)


def shells(Nmesh, BoxSize, kedges):
    """shell index of every mode of the compressed half, -1 for none"""
    kx, ky, kz = po.k_coords(Nmesh, BoxSize, coord_dtype="f4")
    k2 = (kx ** 2 + ky ** 2) + kz ** 2                      # float32, as the reference's sum(xi ** 2) associates it
    dig = np.digitize(k2.astype("f8"), np.asarray(kedges, dtype="f8") ** 2)
    sh = dig - 1
    sh[(dig < 1) | (dig >= len(kedges))] = -1
    sh[0, 0, 0] = -1
    return sh


def _full_shells(sh, N):
    """shells of the full grid from the compressed half: q and -q share |k|"""
    Nx, Ny, Nz = N
    full = np.empty((Nx, Ny, Nz), dtype=sh.dtype)
    full[:, :, :sh.shape[2]] = sh
    kz = np.arange(sh.shape[2], Nz)
    if len(kz):
        mx = (-np.arange(Nx)) % Nx
        my = (-np.arange(Ny)) % Ny
        full[:, :, kz] = sh[mx[:, None, None], my[None, :, None], (Nz - kz)[None, None, :]]
    return full


def _table(kedges, tri, S, Tsum, volume, Ncells):
    count = np.rint(Tsum / Ncells).astype("i8")
    with np.errstate(invalid="ignore", divide="ignore"):
        B = np.where(count > 0, volume ** 2 * S / Tsum, np.nan)
    return count, B


def fft_form(half, Nmesh, BoxSize, kedges):
    """the estimator of the contract in float64; also `bound` = V^2 sum |I_i||I_j||I_l| / sum J J J per triple"""
    N = tuple(int(v) for v in np.asarray(Nmesh) * np.ones(3, dtype="i8"))
    L = np.asarray(BoxSize, dtype="f8") * np.ones(3)
    V = float(np.prod(L))
    Ncells = float(np.prod(N))
    half = np.asarray(half).astype("c16")
    sh = shells(N, L, kedges)
    n = len(kedges) - 1
    I = [np.fft.irfftn(np.where(sh == s, half, 0), s=N, axes=(0, 1, 2)) * Ncells for s in range(n)]
    J = [np.fft.irfftn((sh == s).astype("c16"), s=N, axes=(0, 1, 2)) * Ncells for s in range(n)]
    tri = triples(kedges)
    S = np.array([np.sum(I[i] * I[j] * I[l]) for i, j, l in tri])
    A = np.array([np.sum(np.abs(I[i] * I[j] * I[l])) for i, j, l in tri])
    Tsum = np.array([np.sum(J[i] * J[j] * J[l]) for i, j, l in tri])
    count, B = _table(kedges, tri, S, Tsum, V, Ncells)
    with np.errstate(invalid="ignore", divide="ignore"):
        bound = np.where(count > 0, V ** 2 * A / Tsum, 0.)
    return dict(triples=tri, S=S, Tsum=Tsum, triangles=count, B=B, bound=bound)


def direct_form(half, Nmesh, BoxSize, kedges):
    """the same B and triangle counts from a direct sum over closed triangles of the full grid (no FFT of the shells)"""
    N = tuple(int(v) for v in np.asarray(Nmesh) * np.ones(3, dtype="i8"))
    L = np.asarray(BoxSize, dtype="f8") * np.ones(3)
    V = float(np.prod(L))
    half = np.asarray(half).astype("c16")
    Ncells = float(np.prod(N))
    # the full spectrum of the real field whose half is `half` (what the c2r of the estimator sees)
    c = np.fft.fftn(np.fft.irfftn(half, s=N, axes=(0, 1, 2)))
    sh = _full_shells(shells(N, L, kedges), N)
    n = len(kedges) - 1
    members = [np.argwhere(sh == s) for s in range(n)]
    Nv = np.array(N)
    S3 = {}
    T3 = {}
    for i in range(n):
        for j in range(i, n):
            q1, q2 = members[i], members[j]
            if len(q1) == 0 or len(q2) == 0:
                continue
            q3 = (-(q1[:, None, :] + q2[None, :, :])) % Nv
            s3 = sh[q3[..., 0], q3[..., 1], q3[..., 2]]
            val = (c[q1[:, 0], q1[:, 1], q1[:, 2]][:, None] * c[q2[:, 0], q2[:, 1], q2[:, 2]][None, :]
                   * c[q3[..., 0], q3[..., 1], q3[..., 2]])
            ok = s3 >= 0
            S3[i, j] = np.bincount(s3[ok], weights=val[ok].real, minlength=n)
            T3[i, j] = np.bincount(s3[ok], minlength=n)
    tri = triples(kedges)
    S = np.array([S3[i, j][l] if (i, j) in S3 else 0. for i, j, l in tri])
    count = np.array([T3[i, j][l] if (i, j) in T3 else 0 for i, j, l in tri], dtype="i8")
    with np.errstate(invalid="ignore", divide="ignore"):
        B = np.where(count > 0, V ** 2 * S / count, np.nan)
    return dict(triples=tri, S=S * Ncells, Tsum=count * Ncells, triangles=count, B=B)
