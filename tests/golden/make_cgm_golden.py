"""
Regenerate tests/golden/cgm_*.npz: inputs of CylindricalGroups and the output of the reference's own `cgm()` on them
(nbodykit/algorithms/cgm.py, run verbatim on one rank by oracle/cgm_refload.py), checked here against the reference
test's `direct_cgm` where that applies (flat sky along z).  Needs the reference tree; the fixtures let GPU machines
compare against the reference without it.

    python tests/golden/make_cgm_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import cgm_oracle as co, cgm_refload as cr  # noqa: E402


def cases():
    """name -> (pos, mass, gal_type, rperp, rpar, los or None, periodic, box): the reference test's catalogue (uniform,
    n = 3e-4, log-mass uniform in [12, 15], gal_type from the log-mass) in a smaller box, and a survey-like shell"""
    out = {}
    rng = np.random.RandomState(42)
    L = 160.
    n = int(3e-4 * L ** 3)
    pos = rng.uniform(size=(n, 3)) * L
    logm = rng.uniform(12, 15, size=n)
    gal = np.where(logm < 14.5, 0., 1.)
    out["periodic"] = (pos, 10 ** logm, gal, 10., 10., np.array([0., 0., 1.]), True, L)
    out["nonperiodic"] = (pos, 10 ** logm, gal, 10., 10., np.array([0., 0., 1.]), False, L)
    u = rng.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1)[:, None]
    shell = u * rng.uniform(200., 230., size=n)[:, None]
    out["observer"] = (shell, 10 ** logm, gal, 6., 15., None, False, L)
    return out


def main():
    for name, (pos, mass, gal, rperp, rpar, los, periodic, L) in cases().items():
        t, h, s, prio = co.cgm(pos, [mass, gal], rperp, rpar, los=los, periodic=periodic, BoxSize=L)
        rt, rh, rs = cr.run_cgm(pos, prio, rperp, rpar, los, np.array([L] * 3) if periodic else None)
        for a, b in ((t, rt), (h, rh), (s, rs)):
            assert np.array_equal(a, b), name
        if los is not None and los[2] == 1:
            dn, dt, dh = cr.load().direct_cgm(pos, mass, gal, rperp, rpar, periodic=periodic, BoxSize=[L] * 3)
            assert np.array_equal(dn, rs) and np.array_equal(dt, rt) and np.array_equal(dh, rh), name
        np.savez_compressed(os.path.join(HERE, "cgm_%s.npz" % name), pos=pos, mass=mass, gal_type=gal,
                            rperp=rperp, rpar=rpar, los=np.zeros(0) if los is None else los, periodic=periodic, box=L,
                            cgm_type=rt.astype("u4"), cgm_haloid=rh.astype("i8"), num_cgm_sats=rs.astype("i8"))
        print(name, len(pos), "rows,", int((rt == 1).sum()), "satellites")


if __name__ == "__main__":
    main()
