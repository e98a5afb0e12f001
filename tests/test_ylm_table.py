"""
The real spherical harmonics table the device evaluates (csrc/ylm_table.inc, written by tools/gen_ylm.py with the
reference's sympy recipe) for every (l, m) with l <= 8: the C table equals the JSON copy the oracle evaluates term for
term, and both equal the values of the reference's own get_real_Ylm (tests/golden/ylm_reference.npz, including the
origin, where the polynomial form decides the value) and the real form of scipy.special.sph_harm_y.  CPU only.
"""
import json
import os
import re

import numpy as np
import pytest

from oracle import convpower_oracle as co

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LMAX = 8
LM = [(l, m) for l in range(LMAX + 1) for m in range(-l, l + 1)]


def _inc():
    """(NBK_YLM_LMAX, terms [[c, px, py, pz], ...], offsets [[first, count], ...]) parsed from ylm_table.inc"""
    src = open(os.path.join(ROOT, "nbodykit_b200", "csrc", "ylm_table.inc")).read()
    lmax = int(re.search(r"#define NBK_YLM_LMAX (\d+)", src).group(1))
    terms_src = re.search(r"c_ylm_terms\[(\d+)\] = \{(.*?)\n\};", src, re.S)
    terms = [[float(c), int(a), int(b), int(d)] for c, a, b, d in
             re.findall(r"\{([-+0-9.eE]+), (\d+), (\d+), (\d+)\}", terms_src.group(2))]
    assert len(terms) == int(terms_src.group(1))
    offs_src = re.search(r"c_ylm_off\[(\d+)\]\[2\] = \{(.*?)\n\};", src, re.S)
    offs = [[int(a), int(b)] for a, b in re.findall(r"\{(\d+), (\d+)\}", offs_src.group(2))]
    assert len(offs) == int(offs_src.group(1))
    return lmax, terms, offs


def _golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "ylm_reference.npz"))


def _sph_real(l, m, v):
    """the reference's real Y_lm from scipy's complex one: sympy's assoc_legendre and scipy's P_l^m both carry the
    Condon-Shortley phase, so Y_lm = (-1)^m sqrt(2) Re / Im Y_l^|m| for m > 0 / m < 0"""
    from scipy.special import sph_harm_y
    theta = np.arccos(np.clip(v[:, 2], -1.0, 1.0))
    phi = np.arctan2(v[:, 1], v[:, 0])
    y = sph_harm_y(l, abs(m), theta, phi)
    if m == 0:
        return y.real
    return (-1.0) ** m * np.sqrt(2.0) * (y.real if m > 0 else y.imag)


def test_inc_equals_json():
    """the C table and the oracle's JSON copy are the same polynomials, coefficient for coefficient"""
    lmax, terms, offs = _inc()
    table = json.load(open(os.path.join(ROOT, "tests", "golden", "ylm_table.json")))
    assert lmax == LMAX and table["lmax"] == LMAX
    assert len(offs) == len(LM) == len(table["terms"])
    for l, m in LM:
        first, n = offs[l * l + m + l]
        assert terms[first:first + n] == table["terms"]["%d,%d" % (l, m)], (l, m)
    assert offs[-1][0] + offs[-1][1] == len(terms)


def test_python_limit_matches_table():
    """ConvolvedFFTPower's early check of l uses the table's limit"""
    from nbodykit_b200.algorithms.convpower.fkp import YLM_LMAX
    assert YLM_LMAX == _inc()[0]


def test_golden_covers_table():
    """the reference's get_real_Ylm was sampled for every (l, m) of the table; the l <= 4 values predate the others"""
    g = _golden()
    assert sorted(g.files) == sorted(["vec"] + ["Y_%d_%d" % lm for lm in LM] + ["Y0_%d_%d" % lm for lm in LM])


@pytest.mark.parametrize("l", range(LMAX + 1))
def test_table_vs_reference_values(l):
    """every (l, m): the table against the reference's get_real_Ylm on 64 seeded unit vectors and at the origin"""
    g = _golden()
    v = g["vec"]
    for m in range(-l, l + 1):
        got = co.real_ylm(l, m, v[:, 0], v[:, 1], v[:, 2]) * np.ones(len(v))
        np.testing.assert_allclose(got, g["Y_%d_%d" % (l, m)], rtol=1e-12, atol=1e-12, err_msg="l=%d m=%d" % (l, m))
        # k = 0 has khat := 0: only the constant term survives
        assert abs(float(co.real_ylm(l, m, 0., 0., 0.)) - float(g["Y0_%d_%d" % (l, m)])) < 1e-14, (l, m)


@pytest.mark.parametrize("l", range(LMAX + 1))
def test_table_vs_scipy(l):
    """every (l, m): the table against the real form of scipy.special.sph_harm_y at 10^4 directions and the six
    +-axes, where x^2 + y^2 = 0 leaves phi undefined"""
    rng = np.random.RandomState(100 + l)
    v = rng.standard_normal((10000, 3))
    v /= np.sqrt((v ** 2).sum(axis=1))[:, None]
    v = np.concatenate([v, np.eye(3), -np.eye(3)])
    for m in range(-l, l + 1):
        got = co.real_ylm(l, m, v[:, 0], v[:, 1], v[:, 2]) * np.ones(len(v))
        np.testing.assert_allclose(got, _sph_real(l, m, v), rtol=0, atol=1e-13, err_msg="l=%d m=%d" % (l, m))
