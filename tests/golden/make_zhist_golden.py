"""
Regenerate tests/golden/zhist_*.npz and tests/golden/zhist_reference_save.json: redshifts, weights, and the bin edges,
nbar and interpolation of the reference's own RedshiftHistogram (nbodykit/algorithms/zhist.py, run verbatim on one rank
by oracle/zhist_refload.py), checked here against the restatement of oracle/zhist_oracle.py; and a file written by the
reference's `save`.  Needs the reference tree; the fixtures let GPU machines compare against the reference without it.

    python tests/golden/make_zhist_golden.py
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import zhist_oracle as zo, zhist_refload as zr  # noqa: E402

FSKY = 0.15
EXTS = ("extrapolate", "zeros", "const")


def cases():
    """name -> (z, w, bins): the reference test's N(0.5, 0.1) draw (1000 rows, seed 42) under Scott's rule, and rows on
    every interior edge, on the last edge, below the first edge and NaN under non-uniform explicit edges"""
    out = {}
    z = zo.make_redshifts(42, 1000)
    w = np.random.RandomState(7).uniform(size=z.size)
    out["scott"] = (z, w, None)
    edges = np.array([0.1, 0.2, 0.25, 0.4, 0.45, 0.5, 0.55, 0.62, 0.8, 1.0])
    rng = np.random.RandomState(8)
    ze = np.concatenate([rng.uniform(0.05, 1.05, 800), edges, edges[1:-1], [edges[-1]] * 3, [0.0, 0.09999, np.nan, np.nan]])
    out["explicit"] = (ze, rng.uniform(size=ze.size), edges)
    return out


def probe(centers):
    """interpolation points: a grid over and beyond the centers, the centers and the midpoints between them"""
    lo, hi = centers[0], centers[-1]
    span = hi - lo
    return np.concatenate([np.linspace(lo - 0.2 * span, hi + 0.2 * span, 301), centers, 0.5 * (centers[1:] + centers[:-1])])


def main():
    from nbodykit_b200.cosmology import Planck15
    cosmo = zr.CosmoDict(Planck15)
    for name, (z, w, bins) in cases().items():
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            r = zr.run(z, FSKY, cosmo, bins=bins)
            rw = zr.run(z, FSKY, cosmo, bins=bins, w=w)
            o = zo.zhist(z, FSKY, Planck15, bins=bins)
            ow = zo.zhist(z, FSKY, Planck15, bins=bins, w=w)
        assert np.array_equal(r.bin_edges, o["bin_edges"]) and np.array_equal(r.nbar, o["nbar"]), name
        assert np.array_equal(rw.nbar, ow["nbar"]), name
        x = probe(r.bin_centers)
        interp = {"interp_%s" % e: r.interpolate(x, e) for e in EXTS}
        for e in EXTS:
            assert np.array_equal(interp["interp_%s" % e], zo.interpolate(x, o["bin_centers"], o["nbar"], e)), (name, e)
        np.savez_compressed(os.path.join(HERE, "zhist_%s.npz" % name), z=z, w=w, fsky=np.float64(FSKY),
                            bin_edges=r.bin_edges, bin_centers=r.bin_centers, dV=r.dV, nbar=r.nbar, nbar_weighted=rw.nbar,
                            x=x, **interp)
        if name == "scott":
            r.save(os.path.join(HERE, "zhist_reference_save.json"))
        print(name, len(z), "rows,", len(r.bin_edges) - 1, "bins")


if __name__ == "__main__":
    main()
