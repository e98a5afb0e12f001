// A cubic B-spline (t, c) at x, as FITPACK's splev evaluates it: the knot interval l (t[l] <= x < t[l+1], clamped to
// [k, nt - k - 2], so that x outside [t[k], t[nt-k-1]] is extrapolated with the end polynomial pieces) and the de Boor-Cox
// recurrence of fpbspl.  Shared by the n(z) spline (zhist.cu) and the stellar-to-halo-mass spline of the HOD (hod.cu); both
// files are compiled with --fmad=false, so the value rounds as FITPACK's compiled without contraction does.
#pragma once

#define NBK_SPLEV_K 3          // spline degree

static __device__ __forceinline__ double nbk_splev3(double x, const double *__restrict__ t, int nt,
                                                    const double *__restrict__ c) {
    int lo = NBK_SPLEV_K, hi = nt - NBK_SPLEV_K - 1;   // the largest l in [k, nt - k - 2] with t[l] <= x (k when none)
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(t + mid) <= x) lo = mid;
        else hi = mid;
    }
    const int l = lo;
    double h[NBK_SPLEV_K + 1], hh[NBK_SPLEV_K];
    h[0] = 1.0;
#pragma unroll
    for (int j = 1; j <= NBK_SPLEV_K; j++) {
#pragma unroll
        for (int i = 0; i < j; i++) hh[i] = h[i];
        h[0] = 0.0;
#pragma unroll
        for (int i = 1; i <= j; i++) {
            const double tli = __ldg(t + l + i), tlj = __ldg(t + l + i - j);
            if (tli == tlj) {
                h[i] = 0.0;
                continue;
            }
            const double f = hh[i - 1] / (tli - tlj);
            h[i - 1] = h[i - 1] + f * (tli - x);
            h[i] = f * (x - tlj);
        }
    }
    double sp = 0.0;
#pragma unroll
    for (int j = 0; j <= NBK_SPLEV_K; j++) sp = sp + __ldg(c + l - NBK_SPLEV_K + j) * h[j];
    return sp;
}
