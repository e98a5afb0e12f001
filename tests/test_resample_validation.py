"""Fourier-space resampling without a GPU: the row plan of the P > 1 exchange against a brute-force label match, and
argument validation of the resample entry points (every rejected call returns -1 with a message before any CUDA call)."""
import numpy as np
import pytest

from nbodykit_b200 import _lib


def _freq(i, n):
    return i if i < (n + 1) // 2 else i - n


def _brute_plan(ns, nd, P):
    """{(s, d): {destination row: source row}} by matching labels row by row"""
    m = min(ns, nd)
    out = {}
    for i in range(nd):
        j = _freq(i, nd)
        if -m <= 2 * j < m:
            src = j % ns
            out.setdefault((src // (ns // P), i // (nd // P)), {})[i] = src
    return out


CASES = [(ns, nd, P) for P in (1, 2, 3, 4, 5, 8)
         for ns in (P * k for k in (1, 2, 3, 7, 11, 16))
         for nd in (P * k for k in (1, 2, 5, 8, 9, 12))
         if ns >= 2 and nd >= 2]


@pytest.mark.parametrize("ns,nd,P", CASES)
def test_resample_row_plan_matches_brute_force(ns, nd, P):
    from nbodykit_b200.pmesh.pm import resample_row_plan
    plan = resample_row_plan(ns, nd, P)
    want = _brute_plan(ns, nd, P)
    got = {}
    for s in range(P):
        for d in range(P):
            ranges = plan[s][d]
            assert len(ranges) <= 2
            assert [r[0] for r in ranges] == sorted(r[0] for r in ranges)
            for d0, s0, n in ranges:
                assert n > 0
                for t in range(n):
                    assert (d0 + t) // (nd // P) == d and (s0 + t) // (ns // P) == s
                    got.setdefault((s, d), {})[d0 + t] = s0 + t
    assert got == want


def test_resample_row_plan_examples():
    from nbodykit_b200.pmesh.pm import resample_row_plan
    # 32 -> 48 on one rank: labels 0..15 and -16..-1 (the source Nyquist row 16 goes to label -16, row 32)
    assert resample_row_plan(32, 48, 1) == [[[(0, 0, 16), (32, 16, 16)]]]
    # 45 -> 33 on three ranks of 15 / 11 rows: labels 0..16 and -16..-1
    plan = resample_row_plan(45, 33, 3)
    assert plan[0][0] == [(0, 0, 11)] and plan[0][1] == [(11, 11, 4)] and plan[0][2] == []
    assert plan[1][1] == [(15, 15, 2), (17, 29, 1)] and plan[1][2] == []          # two ranges: the labels wrap
    assert plan[2][1] == [(18, 30, 4)] and plan[2][2] == [(22, 34, 11)]


def test_resample_entry_points_reject_bad_arguments():
    L = _lib.lib()
    a, b = _lib.iarr([8, 8, 8]), _lib.iarr([12, 12, 12])
    assert L.nbk_resample_complex(None, None, 3, a, b, None) == -1 and b"dtype" in L.nbk_last_error()
    assert L.nbk_resample_complex(None, None, 8, a, b, None) == -1 and b"buffers" in L.nbk_last_error()
    assert L.nbk_resample_pack(None, None, 3, a, b, 4, _lib.iarr([0, 1]), 1, None) == -1 and b"dtype" in L.nbk_last_error()
    assert L.nbk_resample_pack(None, None, 8, a, _lib.iarr([12, 12, 1]), 4, _lib.iarr([0, 1]), 1, None) == -1
    assert b"2 .. 2^24" in L.nbk_last_error()
    assert L.nbk_resample_pack(None, None, 8, a, b, 9, _lib.iarr([0, 1]), 1, None) == -1 and b"local rows" in L.nbk_last_error()
    assert L.nbk_resample_pack(None, None, 8, a, b, 4, _lib.iarr([3, 2]), 1, None) == -1 and b"outside" in L.nbk_last_error()
    assert L.nbk_resample_pack(None, None, 8, a, b, 4, _lib.iarr([-1, 1]), 1, None) == -1 and b"outside" in L.nbk_last_error()
    assert L.nbk_resample_pack(None, None, 8, a, b, 4, _lib.iarr([0] * 66), 33, None) == -1 and b"at most 32" in L.nbk_last_error()
    assert L.nbk_resample_pack(None, None, 8, a, b, 4, _lib.iarr([0, 1]), 1, None) == -1 and b"buffers" in L.nbk_last_error()
    assert L.nbk_resample_unpack(None, None, 4, b, 4, _lib.iarr([0, 1]), 1, None) == -1 and b"buffers" in L.nbk_last_error()
    assert L.nbk_resample_unpack(None, None, 8, b, 4, _lib.iarr([0, 2, 1, 2]), 2, None) == -1
    assert b"overlap" in L.nbk_last_error()
    assert L.nbk_resample_unpack(None, None, 8, b, 13, _lib.iarr([]), 0, None) == -1 and b"local rows" in L.nbk_last_error()


def test_resample_entry_points_with_nothing_to_do_need_no_gpu():
    L = _lib.lib()
    a, b = _lib.iarr([8, 8, 8]), _lib.iarr([12, 12, 12])
    assert L.nbk_resample_pack(None, None, 8, a, b, 4, _lib.iarr([0, 0, 2, 0]), 2, None) == 0
    assert L.nbk_resample_pack(None, None, 4, a, b, 0, _lib.iarr([]), 0, None) == 0
    assert L.nbk_resample_unpack(None, None, 8, b, 0, _lib.iarr([]), 0, None) == 0


def test_version_bumped_for_the_resample_exchange():
    assert _lib.lib().nbk_version() >= 104


def test_preview_at_a_size_not_divisible_by_the_ranks_raises_before_any_gpu_work():
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.pmesh.pm import ParticleMesh, RealField

    class Fake(SelfComm):
        def __init__(self, rank, size):
            self.rank, self.size = rank, size
    pm = ParticleMesh(BoxSize=1., Nmesh=[12, 12, 8], dtype='f8', comm=Fake(0, 3))
    f = RealField.__new__(RealField)
    f.pm = pm
    with pytest.raises(ValueError, match="divisible by the number of GPUs"):
        f.preview(Nmesh=[8, 9, 8], axes=(0, 1))
    np.testing.assert_array_equal(pm.Nmesh, [12, 12, 8])
