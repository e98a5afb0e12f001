"""
TEST INFRASTRUCTURE -- float64 NumPy oracle for ConvolvedFFTBispectrum (nbodykit_b200/algorithms/convbispectrum.py,
DESIGN.md 4.15).  NOT product code.  Fields F and N come from oracle.convpower_oracle.fkp_field's paint (fkp_fields) or
from the caller; shells, triples and rows are those of oracle/bispectrum_oracle.py and bispectrum_poles_oracle.py.

Inputs: F (the FKP field), N (the shot field: mass u^2, +alpha^2 for the randoms, / V_cell), the compensation name or
None, I33 and S3.  x_hat is the unit vector of the cell coordinates (convpower_oracle.x_coords) + BoxCenter + H / 2,
q_hat that of the wavenumber coordinates (pmesh_oracle.k_coords), and the compensation takes the circular coordinates,
all in `coord_dtype` (float64 by default, the arithmetic of the Y_lm and compensation kernels); the shells are decided
at float32 coordinates as FFTPower's k bins.

  fft_form    -- the contract: c = r2c(F), G_ell = 4 pi sum_m Y_lm(q_hat) r2c[F Y_lm(x_hat)] (compensated), I, W, J, H by
                 irfftn of the shell-masked half spectra; B_ell = V^3 sum W_a I_b I_c / (I33 sum J J J) per row and
                 shotnoise_0 per sorted triple; `bound` = V^3 sum |W_a||I_b||I_c| / (I33 sum J J J) and `shot_bound`
  direct_form -- no Y_lm and no FFT of the shells: G_ell(q) = (2 ell + 1) sum_x F(x) L_ell(q_hat.x_hat) e^{-i q.x} / N^3
                 summed explicitly on the full grid, projected to what a c2r of its stored half represents, and closed
                 triangles q1 + q2 + q3 = 0 (modulo the grid) enumerated.  Meshes of 16^3 cells or fewer.
"""
import numpy as np

from oracle import bispectrum_oracle as bo
from oracle import convpower_oracle as co
from oracle import pmesh_oracle as po

import bispectrum_poles_oracle as bpo


def fkp_fields(dpos, rpos, d, r, Nmesh, BoxSize, BoxCenter, resampler="cic", dtype="f8"):
    """F, N, alpha, data.norm3, randoms.norm3 and S3 of catalogues given as dicts of float64 columns wc, wf, nbar, v
    (F through convpower_oracle.fkp_field; N with mass u^2 = (wc wf v)^2 and +alpha^2 for the randoms)"""
    N3 = np.asarray(Nmesh, dtype="i8") * np.ones(3, dtype="i8")
    L = np.asarray(BoxSize, dtype="f8") * np.ones(3)
    C = np.asarray(BoxCenter, dtype="f8") * np.ones(3)
    F, alpha = co.fkp_field(dpos, rpos, (d["wc"], d["wf"] * d["v"]), (r["wc"], r["wf"] * r["v"]), N3, L, C, resampler,
                            dtype)
    ud, ur = d["wc"] * d["wf"] * d["v"], r["wc"] * r["wf"] * r["v"]
    Nf = (po.paint(dpos - C, ud ** 2, N3, L, resampler) + alpha ** 2 * po.paint(rpos - C, ur ** 2, N3, L, resampler))
    Nf = (Nf / (L / N3).prod()).astype(dtype)
    norm_d = float((d["nbar"] ** 2 * d["wc"] * d["wf"] ** 3).sum())
    norm_r = alpha * float((r["nbar"] ** 2 * r["wc"] * r["wf"] ** 3).sum())
    S3 = float((ud ** 3).sum()) - alpha ** 3 * float((ur ** 3).sum())
    return dict(F=F, N=Nf, alpha=alpha, data_norm3=norm_d, randoms_norm3=norm_r, S3=S3)


def _geom(Nmesh, BoxSize):
    N = tuple(int(v) for v in np.asarray(Nmesh, dtype="i8") * np.ones(3, dtype="i8"))
    L = np.asarray(BoxSize, dtype="f8") * np.ones(3)
    return N, L, float(np.prod(L)), float(np.prod(N))


def _unit(vs):
    n = np.sqrt(sum(v ** 2 for v in vs))
    n = np.where(n == 0., np.inf, n)
    return [v / n for v in vs]


def _xhat(N, L, BoxCenter, coord_dtype):
    off = np.asarray(BoxCenter, dtype="f8") * np.ones(3) + 0.5 * L / np.array(N)
    return _unit([x.astype("f8") + off[i] for i, x in enumerate(co.x_coords(N, L, coord_dtype))])


def _rows_of(kedges):
    return bo.triples(kedges), bpo.pole_rows(kedges)


def _assemble(kedges, V, Nc, I33, S3, poles, tri, rows, S_rows, A_rows, Tsum_rows, Tsum_tri, H_tri, HA_tri, count_tri):
    """B_ell per row, shotnoise_0 per sorted triple, their bounds and triangle counts"""
    out = dict(triples=tri, rows=rows, triangles=count_tri, Tsum=Tsum_tri)
    idx = {tuple(t): q for q, t in enumerate(tri.tolist())}
    rcount = count_tri[[idx[tuple(sorted(r))] for r in rows.tolist()]] if len(rows) else np.zeros(0, dtype="i8")
    out["row_triangles"] = rcount
    with np.errstate(invalid="ignore", divide="ignore"):
        for ell in poles:
            out["B_%d" % ell] = np.where(rcount > 0, V ** 3 * S_rows[ell] / (I33 * Tsum_rows), np.nan)
            out["bound_%d" % ell] = np.where(rcount > 0, V ** 3 * A_rows[ell] / (I33 * Tsum_rows), 0.)
        if H_tri is not None:
            out["shotnoise_0"] = np.where(count_tri > 0, (H_tri / Tsum_tri - 2 * S3) / I33, np.nan)
            out["shot_bound"] = np.where(count_tri > 0, (HA_tri / Tsum_tri + 2 * abs(S3)) / abs(I33), 0.)
    return out


def fft_form(F, Nf, Nmesh, BoxSize, BoxCenter, kedges, poles, comp, I33, S3, coord_dtype="f8"):
    N, L, V, Nc = _geom(Nmesh, BoxSize)
    F = np.asarray(F, dtype="f8")
    wc = po.k_coords(N, L, coord_dtype, kind="circular")
    cm = (lambda v: po.compensate(comp, wc, v)) if comp else (lambda v: v)      # noqa: E731
    c = cm(po.r2c(F))
    xh = _xhat(N, L, BoxCenter, coord_dtype)
    kh = _unit([k.astype("f8") for k in po.k_coords(N, L, coord_dtype)])
    G = {0: c}
    for ell in [l for l in poles if l > 0]:
        acc = np.zeros_like(c)
        for m in range(-ell, ell + 1):
            acc += po.r2c(F * co.real_ylm(ell, m, *xh)) * co.real_ylm(ell, m, *kh)
        G[ell] = cm(4 * np.pi * acc)
    sh = bo.shells(N, L, kedges)
    n = len(kedges) - 1
    c2r = lambda a: np.fft.irfftn(a, s=N, axes=(0, 1, 2)) * Nc             # noqa: E731
    W = {ell: [c2r(np.where(sh == s, G[ell], 0)) for s in range(n)] for ell in G}
    I = W[0]
    J = [c2r((sh == s).astype("c16")) for s in range(n)]
    tri, rows = _rows_of(kedges)
    Tsum_tri = np.array([np.sum(J[i] * J[j] * J[l]) for i, j, l in tri])
    Tsum_rows = np.array([np.sum(J[a] * J[b] * J[cc]) for a, b, cc in rows])
    S = {ell: np.array([np.sum(W[ell][a] * I[b] * I[cc]) for a, b, cc in rows]) for ell in poles}
    A = {ell: np.array([np.sum(np.abs(W[ell][a] * I[b] * I[cc])) for a, b, cc in rows]) for ell in poles}
    H_tri = HA_tri = None
    if 0 in poles:
        cN = cm(po.r2c(np.asarray(Nf, dtype="f8")))
        H = [c2r(np.where(sh == s, V * V * c * np.conj(cN), 0)) for s in range(n)]
        H_tri = np.array([np.sum(H[i] * J[j] * J[l] + J[i] * H[j] * J[l] + J[i] * J[j] * H[l]) for i, j, l in tri])
        HA_tri = np.array([np.sum(np.abs(H[i] * J[j] * J[l]) + np.abs(J[i] * H[j] * J[l]) + np.abs(J[i] * J[j] * H[l]))
                           for i, j, l in tri])
    count = np.rint(Tsum_tri / Nc).astype("i8")
    return _assemble(kedges, V, Nc, I33, S3, poles, tri, rows, S, A, Tsum_rows, Tsum_tri, H_tri, HA_tri, count)


def _full_coords(N, L, coord_dtype, kind):
    ct = np.dtype(coord_dtype).type
    out = []
    for d in range(3):
        j = po.freq_index(N[d])
        unit = (2 * np.pi / L[d]) if kind == "wavenumber" else (2 * np.pi / N[d])
        shape = [1, 1, 1]
        shape[d] = N[d]
        out.append((j.astype(ct) * ct(unit)).reshape(shape))
    return out


def _half_projection(G, N):
    """what the c2r of G's stored half (kz <= Nz // 2) represents on the full grid: G where stored, conj(G(-q)) at the
    mirror of a stored mode, the mean of the two on the planes that are their own mirror (kz = 0, kz = Nz / 2)"""
    m = [(-np.arange(n)) % n for n in N]
    Gm = np.conj(G[m[0][:, None, None], m[1][None, :, None], m[2][None, None, :]])
    kz = np.arange(N[2])[None, None, :]
    self_mirror = (kz == 0) | (2 * kz == N[2])
    return np.where(self_mirror, 0.5 * (G + Gm), np.where(kz <= N[2] // 2, G, Gm))


def direct_form(F, Nf, Nmesh, BoxSize, BoxCenter, kedges, poles, comp, I33, S3, coord_dtype="f8"):
    N, L, V, Nc = _geom(Nmesh, BoxSize)
    assert Nc <= 16 ** 3, "the direct form sums every cell for every mode: 16^3 cells at most"
    F = np.asarray(F, dtype="f8").reshape(-1)
    kf = _full_coords(N, L, coord_dtype, "wavenumber")
    wc = _full_coords(N, L, coord_dtype, "circular")
    cm = (lambda v: po.compensate(comp, wc, v)) if comp else (lambda v: v)      # noqa: E731
    xh = [np.broadcast_to(x, N).reshape(-1) for x in _xhat(N, L, BoxCenter, coord_dtype)]
    kh = [np.broadcast_to(k, N).reshape(-1) for k in _unit([k.astype("f8") for k in kf])]
    # e^{-i q.x} with the integer labels: q.x = 2 pi sum_d j_d i_d / N_d
    ji = np.indices(N).reshape(3, -1)
    jq = [np.broadcast_to(po.freq_index(N[d]).reshape([-1 if e == d else 1 for e in range(3)]), N).reshape(-1)
          for d in range(3)]
    G = {}
    ells = sorted(set([0] + list(poles)))
    nq = len(jq[0])
    acc = {ell: np.zeros(nq, dtype="c16") for ell in ells}
    for q0 in range(0, nq, 256):
        q1 = min(q0 + 256, nq)
        ph = sum(np.outer(jq[d][q0:q1], ji[d]) / N[d] for d in range(3))
        e = np.exp(-2j * np.pi * ph) * F[None, :]
        mu = sum(np.outer(kh[d][q0:q1], xh[d]) for d in range(3))
        for ell in ells:
            acc[ell][q0:q1] = (e * bpo.legendre(ell, mu)).sum(axis=1)
    for ell in ells:
        G[ell] = _half_projection(cm((2 * ell + 1) * acc[ell].reshape(N) / Nc), N)
    c = G[0]
    sh = bo._full_shells(bo.shells(N, L, kedges), N)
    n = len(kedges) - 1
    members = [np.argwhere(sh == s) for s in range(n)]
    Nv = np.array(N)
    h = None
    if 0 in poles:
        Fn = np.asarray(Nf, dtype="f8").reshape(-1)
        cN = np.zeros(nq, dtype="c16")
        for q0 in range(0, nq, 256):
            q1 = min(q0 + 256, nq)
            ph = sum(np.outer(jq[d][q0:q1], ji[d]) / N[d] for d in range(3))
            cN[q0:q1] = (np.exp(-2j * np.pi * ph) * Fn[None, :]).sum(axis=1)
        cN = _half_projection(cm(cN.reshape(N) / Nc), N)
        h = V * V * c * np.conj(cN)
    S3d, T3, H3 = {}, {}, {}
    for a in range(n):
        for b in range(n):
            qa, qb = members[a], members[b]
            if len(qa) == 0 or len(qb) == 0:
                continue
            qc = (-(qa[:, None, :] + qb[None, :, :])) % Nv
            sc = sh[qc[..., 0], qc[..., 1], qc[..., 2]]
            ok = sc >= 0
            T3[a, b] = np.bincount(sc[ok], minlength=n)
            cc = c[qb[:, 0], qb[:, 1], qb[:, 2]][None, :] * c[qc[..., 0], qc[..., 1], qc[..., 2]]
            for ell in poles:
                val = G[ell][qa[:, 0], qa[:, 1], qa[:, 2]][:, None] * cc
                S3d[ell, a, b] = np.bincount(sc[ok], weights=val[ok].real, minlength=n)
            if h is not None:
                hv = (h[qa[:, 0], qa[:, 1], qa[:, 2]][:, None] + h[qb[:, 0], qb[:, 1], qb[:, 2]][None, :]
                      + h[qc[..., 0], qc[..., 1], qc[..., 2]])
                H3[a, b] = np.bincount(sc[ok], weights=hv[ok].real, minlength=n)
    tri, rows = _rows_of(kedges)
    count = np.array([T3[i, j][l] if (i, j) in T3 else 0 for i, j, l in tri], dtype="i8")
    rcount = np.array([T3[a, b][cc] if (a, b) in T3 else 0 for a, b, cc in rows], dtype="i8")
    S = {ell: np.array([S3d[ell, a, b][cc] if (ell, a, b) in S3d else 0. for a, b, cc in rows]) * Nc for ell in poles}
    A = {ell: np.abs(S[ell]) for ell in poles}
    H_tri = None
    if h is not None:
        H_tri = np.array([H3[i, j][l] if (i, j) in H3 else 0. for i, j, l in tri]) * Nc
    return _assemble(kedges, V, Nc, I33, S3, poles, tri, rows, S, A, rcount * Nc, count * Nc, H_tri,
                     None if H_tri is None else np.abs(H_tri), count)
