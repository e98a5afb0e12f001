"""
Float64 NumPy/SciPy restatement of the Zheng07 population of DESIGN.md 4.13 (HaloCatalog.populate), with the same
counter-based draws as csrc/hod.cu, for the tests.

populate(mass, radius, conc, pos, vel, box, params, seed, ...) returns the galaxy columns of one rank whose halos are
the global rows h0 .. h0 + n - 1, in the kernels' row order (centrals in halo order, then satellites in (halo, k) order).
The NFW radius inverse, the Jeans table and the samplers are written out here, separately from the package.
"""
import math

import numpy
from scipy.special import erf, gammaln

MASK = (1 << 64) - 1
G_KMS2_MPC_PER_MSUN = 1.3271244e20 / 3.0856775814913673e22 / 1e6     # IAU 2015 GM_sun over the Mpc, in (km/s)^2 Mpc / M_sun


# ---- draws -------------------------------------------------------------------------------------------------------------
def mix(z):
    """SplitMix64 finaliser on uint64 arrays (wrapping arithmetic)"""
    z = numpy.asarray(z, dtype=numpy.uint64)
    with numpy.errstate(over='ignore'):
        z = z + numpy.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> numpy.uint64(30))) * numpy.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> numpy.uint64(27))) * numpy.uint64(0x94D049BB133111EB)
    return z ^ (z >> numpy.uint64(31))


def key(seed, stream, h):
    """the key of the draws of global halo rows h in `stream`"""
    s = mix(numpy.full(numpy.shape(h), seed, dtype=numpy.uint64))
    return mix(mix(s ^ numpy.uint64(stream)) ^ numpy.asarray(h, dtype=numpy.int64).astype(numpy.uint64))


def uniform(k, j):
    """draw j of keys k: ((x >> 12) + 1/2) 2^-52 in (0, 1)"""
    x = mix(numpy.asarray(k, dtype=numpy.uint64) ^ numpy.asarray(j, dtype=numpy.int64).astype(numpy.uint64))
    return ((x >> numpy.uint64(12)).astype('f8') + 0.5) * 2.0 ** -52


# ---- occupation --------------------------------------------------------------------------------------------------------
def mean_central(m, logMmin, sigma_logM):
    return 0.5 * (1.0 + erf((numpy.log10(m) - logMmin) / sigma_logM))


def mean_satellite(m, logMmin, sigma_logM, logM0, logM1, alpha, modulate=True):
    M0, M1 = 10. ** logM0, 10. ** logM1
    with numpy.errstate(invalid='ignore'):
        lam = numpy.where(m > M0, ((m - M0) / M1) ** alpha, 0.0)
    if modulate:
        lam = lam * mean_central(m, logMmin, sigma_logM)
    return lam


def poisson(k, lam):
    """exact Poisson(lam) from draws 1, 2, ... of keys k: sequential inversion below 10, PTRS (Hormann 1993) above"""
    k = numpy.asarray(k, dtype=numpy.uint64)
    lam = numpy.asarray(lam, dtype='f8')
    out = numpy.zeros(lam.shape, dtype=numpy.int64)
    inv = numpy.flatnonzero((lam > 0) & (lam < 10.0))
    if inv.size:
        L = lam[inv]
        u = uniform(k[inv], 1)
        p = numpy.exp(-L)
        s = p.copy()
        x = numpy.zeros(inv.size, dtype=numpy.int64)
        for _ in range(1000):
            act = u > s
            if not act.any():
                break
            x[act] += 1
            p[act] = p[act] * (L[act] / x[act].astype('f8'))
            s[act] = s[act] + p[act]
        out[inv] = x
    big = numpy.flatnonzero(lam >= 10.0)
    if big.size:
        L = lam[big]
        slam, loglam = numpy.sqrt(L), numpy.log(L)
        b = 0.931 + 2.53 * slam
        a = -0.059 + 0.02483 * b
        invalpha = 1.1239 + 1.1328 / (b - 3.4)
        vr = 0.9277 - 3.6224 / (b - 2.0)
        todo = numpy.arange(big.size)
        j = 1
        while todo.size:
            U = uniform(k[big[todo]], j) - 0.5
            V = uniform(k[big[todo]], j + 1)
            us = 0.5 - numpy.abs(U)
            kk = numpy.floor((2.0 * a[todo] / us + b[todo]) * U + L[todo] + 0.43)
            acc = (us >= 0.07) & (V <= vr[todo])
            rej = ~acc & ((kk < 0) | ((us < 0.013) & (V > us)))
            test = ~acc & ~rej
            with numpy.errstate(invalid='ignore', divide='ignore'):
                lhs = numpy.log(V) + numpy.log(invalpha[todo]) - numpy.log(a[todo] / (us * us) + b[todo])
                rhs = -L[todo] + kk * loglam[todo] - gammaln(kk + 1.0)
            acc = acc | (test & (lhs <= rhs))
            out[big[todo[acc]]] = kk[acc].astype(numpy.int64)
            todo = todo[~acc]
            j += 2
    return out


def occupy(mass, h0, params, seed, modulate=True):
    """(N_cen, N_sat) of the halos of masses `mass` at global rows h0 .."""
    m = numpy.asarray(mass, dtype='f8')
    h = h0 + numpy.arange(m.size, dtype=numpy.int64)
    k = key(seed, 0, h)
    p = mean_central(m, params['logMmin'], params['sigma_logM'])
    lam = mean_satellite(m, params['logMmin'], params['sigma_logM'], params['logM0'], params['logM1'], params['alpha'],
                         modulate)
    ncen = (uniform(k, 0) < p).astype(numpy.int64)
    return ncen, poisson(k, lam)


# ---- NFW profile -------------------------------------------------------------------------------------------------------
def g(y):
    """ln(1 + y) - y / (1 + y), by its series below y = 0.1"""
    y = numpy.asarray(y, dtype='f8')
    s = numpy.zeros_like(y)
    ys = numpy.minimum(y, 0.1)
    for m in range(16, -1, -1):
        s = s * (-ys) + float(m + 1) / float(m + 2)
    with numpy.errstate(invalid='ignore', divide='ignore'):
        big = numpy.log1p(y) - y / (1.0 + y)
    return numpy.where(y < 0.1, ys * ys * s, big)


def ginv(a):
    """y with g(y) = a: -1 - 1 / W0(-exp(-1 - a)), started from the W0 series at the branch point (p < 1) or at 0, and
    finished by four Halley steps on g(y) = a"""
    a = numpy.asarray(a, dtype='f8')
    p = numpy.sqrt(2.0 * -numpy.expm1(-a))
    w = p * (1.0 + p * (-1.0 / 3.0 + p * (11.0 / 72.0 + p * (-43.0 / 540.0 + p * (769.0 / 17280.0)))))
    z = -numpy.exp(-1.0 - a)
    W = z * (1.0 + z * (-1.0 + z * (1.5 + z * (-8.0 / 3.0 + z * (125.0 / 24.0)))))
    with numpy.errstate(divide='ignore', invalid='ignore'):
        y = numpy.where(p < 1.0, w / (1.0 - w), -1.0 - 1.0 / W)
    for _ in range(4):
        q = 1.0 + y
        F = g(y) - a
        F1 = y / (q * q)
        F2 = (1.0 - y) / (q * q * q)
        y = y - (2.0 * F * F1) / (2.0 * F1 * F1 - F * F2)
    return y


S0, HS, K = -20.0, 1.0 / 128, 44 * 128 + 1
_GX, _GW = numpy.polynomial.legendre.leggauss(8)
_TAB = None


def _q(s):
    y = numpy.exp(s)
    return g(y) / (y * y * (1.0 + y) ** 2)


def _panels(a, h, n):
    left = a + numpy.arange(n) * h
    acc = numpy.zeros(n)
    for x, w in zip(_GX, _GW):
        acc += float(w) * _q(left + 0.5 * h * (1.0 + float(x)))
    return 0.5 * h * acc


def jeans_table():
    """(K, 2): ln I and d ln I / ds at s = ln y = S0 + k HS, I(y) = int_y^inf g(t) / (t^3 (1 + t)^2) dt"""
    global _TAB
    if _TAB is None:
        s = S0 + numpy.arange(K) * HS
        tail = _panels(s[-1], HS, int(round((64.0 - s[-1]) / HS))).sum()
        inner = _panels(S0, HS, K - 1)
        I = numpy.empty(K)
        I[-1] = tail
        I[:-1] = tail + numpy.cumsum(inner[::-1])[::-1]
        _TAB = numpy.stack([numpy.log(I), -_q(s) / I], axis=1)
    return _TAB


def jeans_integral(y):
    """I(y): cubic Hermite interpolation of ln I in ln y, with the series at 0 and infinity outside the table"""
    tab = jeans_table()
    y = numpy.asarray(y, dtype='f8')
    s = numpy.log(y)
    s1 = S0 + (K - 1) * HS
    t = (s - S0) / HS
    k = numpy.clip(numpy.floor(numpy.clip(t, 0, K)), 0, K - 2).astype(numpy.int64)
    f = t - k
    f2 = f * f
    f3 = f2 * f
    h00, h10 = 2.0 * f3 - 3.0 * f2 + 1.0, f3 - 2.0 * f2 + f
    h01, h11 = -2.0 * f3 + 3.0 * f2, f3 - f2
    L = h00 * tab[k, 0] + h10 * HS * tab[k, 1] + h01 * tab[k + 1, 0] + h11 * HS * tab[k + 1, 1]
    mid = numpy.exp(L)
    with numpy.errstate(over='ignore', invalid='ignore'):
        low = numpy.exp(tab[0, 0]) + 0.5 * (S0 - s) - (5.0 / 3.0) * (numpy.exp(S0) - y)
        high = numpy.exp(tab[-1, 0]) * ((4.0 * s - 3.0) / (4.0 * s1 - 3.0)) * numpy.exp(-4.0 * (s - s1))
    return numpy.where(s < S0, low, numpy.where(s >= s1, high, mid))


def sigma_r2_over_v2(y, c):
    """sigma_r^2 / V^2 = c / g(c) y (1 + y)^2 I(y)"""
    q = 1.0 + y
    return (c / g(c)) * (y * (q * q)) * jeans_integral(y)


# ---- population --------------------------------------------------------------------------------------------------------
def _wrap(x, L, dtype):
    w = x - L * numpy.floor(x / L)
    w = numpy.where(w >= L, w - L, w)
    w = numpy.where(w < 0, w + L, w)
    o = w.astype(dtype)
    return numpy.where(o.astype('f8') >= L, numpy.zeros((), dtype), o)


def populate(mass, radius, conc, pos, vel, box, params, seed, h0=0, modulate=True, rsd=1.0):
    """the galaxy columns of the halos at global rows h0 .. (one rank), in the kernels' row order; positions and
    velocities of the dtype of `pos` (vel is cast to it first)"""
    mass, radius, conc = [numpy.asarray(a, dtype='f8') for a in (mass, radius, conc)]
    T = numpy.asarray(pos).dtype
    pos = numpy.asarray(pos, dtype=T).reshape(-1, 3)
    vel = numpy.asarray(vel).astype(T).reshape(-1, 3)
    L = numpy.broadcast_to(numpy.asarray(box, dtype='f8'), (3,))
    n = mass.size
    ncen, nsat = occupy(mass, h0, params, seed, modulate)
    ci = numpy.flatnonzero(ncen)
    si = numpy.repeat(numpy.arange(n), nsat)
    sk = numpy.arange(si.size) - numpy.repeat(numpy.cumsum(nsat) - nsat, nsat)
    hidx = numpy.concatenate([ci, si])
    dx = numpy.zeros((hidx.size, 3))
    dv = numpy.zeros((hidx.size, 3))
    r = numpy.zeros(hidx.size)
    if si.size:
        k = key(seed, 1, h0 + si)
        j = 8 * sk
        c, R = conc[si], radius[si]
        gc = g(c)
        y = numpy.minimum(ginv(uniform(k, j) * gc), c)
        rr = (y / c) * R
        mu = 2.0 * uniform(k, j + 1) - 1.0
        phi = 6.283185307179586 * uniform(k, j + 2)
        st = numpy.sqrt(numpy.maximum(0.0, 1.0 - mu * mu))
        q = 1.0 + y
        v2 = G_KMS2_MPC_PER_MSUN * mass[si] / R
        sig = numpy.sqrt(v2 * (c / gc) * (y * (q * q)) * jeans_integral(y))
        r0 = numpy.sqrt(-2.0 * numpy.log(uniform(k, j + 3)))
        t0 = 6.283185307179586 * uniform(k, j + 4)
        r1 = numpy.sqrt(-2.0 * numpy.log(uniform(k, j + 5)))
        t1 = 6.283185307179586 * uniform(k, j + 6)
        ns = ci.size
        dx[ns:] = numpy.stack([rr * (st * numpy.cos(phi)), rr * (st * numpy.sin(phi)), rr * mu], axis=1)
        dv[ns:] = numpy.stack([sig * (r0 * numpy.cos(t0)), sig * (r0 * numpy.sin(t0)), sig * (r1 * numpy.cos(t1))], axis=1)
        r[ns:] = rr
    gpos = numpy.stack([_wrap(pos[hidx, d].astype('f8') + dx[:, d], L[d], T) for d in range(3)], axis=1)
    gvel = (vel[hidx].astype('f8') + dv).astype(T)
    return dict(Position=gpos, Velocity=gvel, VelocityOffset=(gvel.astype('f8') * rsd).astype(T),
                gal_type=numpy.concatenate([numpy.zeros(ci.size, 'i4'), numpy.ones(si.size, 'i4')]),
                halo_id=h0 + hidx, satellite_index=numpy.concatenate([numpy.zeros(ci.size, 'i8'), sk]),
                host_centric_distance=r, ncen=ncen, nsat=nsat)
