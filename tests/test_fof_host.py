"""FOF without a GPU: argument validation of the nbk_fof_* entry points (rejected before any CUDA call), the host-side
errors of FOF / find_features / to_halos, and the CPU restatement in oracle/fof_oracle.py on small cases."""
import ctypes
import os
import sys

import numpy as np
import pytest

from oracle import fof_oracle as fo  # noqa: E402


def test_fof_entry_points_validate_before_cuda():
    from nbodykit_b200 import _lib
    L = _lib.lib()
    box, org, nc = _lib.darr([10., 10., 10.]), _lib.darr([0., 0., 0.]), _lib.iarr([20, 20, 20])
    err = lambda: L.nbk_last_error()  # noqa: E731
    assert L.nbk_fof_cell_keys(None, 3, 10, 1, box, org, nc, 1.0, None, None) == -1 and b"dtype" in err()
    assert L.nbk_fof_cell_keys(None, 4, 1 << 32, 1, box, org, nc, 1.0, None, None) == -1 and b"out of range" in err()
    assert L.nbk_fof_cell_keys(None, 4, 10, 1, box, org, nc, 0.0, None, None) == -1 and b"linking length" in err()
    assert L.nbk_fof_cell_keys(None, 4, 10, 1, box, org, nc, float("nan"), None, None) == -1 and b"linking length" in err()
    assert L.nbk_fof_cell_keys(None, 4, 10, 1, _lib.darr([10., float("inf"), 10.]), org, nc, 1.0, None, None) == -1 \
        and b"finite" in err()
    assert L.nbk_fof_cell_keys(None, 4, 10, 1, box, org, _lib.iarr([20, 0, 20]), 1.0, None, None) == -1 and b"cell count" in err()
    # cells of side 10 / 5 = 2 > 1 / sqrt(3): pairs inside one cell would not all be friends
    assert L.nbk_fof_cell_keys(None, 4, 10, 1, box, org, _lib.iarr([5, 5, 5]), 1.0, None, None) == -1 and b"wider" in err()
    assert L.nbk_fof_cell_keys(None, 4, 10, 0, box, None, nc, 1.0, None, None) == -1 and b"origin" in err()
    assert L.nbk_fof_cell_keys(None, 4, 0, 1, box, org, nc, 1.0, None, None) == 0          # nothing to do
    assert L.nbk_fof_sorted_pos(None, 2, 10, None, 1, box, None, None) == -1 and b"dtype" in err()
    assert L.nbk_fof_compact_count(None, 0, None, 0, None, None) == -1 and b"at least one" in err()
    assert L.nbk_fof_compact_count(None, 10000, None, 2, None, None) == -1 and b"workspace" in err()
    assert L.nbk_fof_compact_write(None, 10000, None, 2, None, None, None) == -1 and b"workspace" in err()
    assert L.nbk_fof_compact_workspace(10000) == 4
    sel = ctypes.c_int(7)
    assert L.nbk_fof_sort(None, None, None, None, 1 << 31, 8, 40, None, 0, ctypes.byref(sel), None) == -1 \
        and b"out of range" in err()
    assert L.nbk_fof_sort(None, None, None, None, 10, 2, 8, None, 0, ctypes.byref(sel), None) == -1 and b"4- or 8-byte" in err()
    assert L.nbk_fof_sort(None, None, None, None, 10, 4, 33, None, 0, ctypes.byref(sel), None) == -1 and b"bit count" in err()
    assert L.nbk_fof_sort(None, None, None, None, 0, 4, 8, None, 0, ctypes.byref(sel), None) == 0 and sel.value == 0
    assert L.nbk_fof_sort_workspace(1000, 3) == -1 and L.nbk_fof_sort_workspace(-1, 8) == -1
    assert L.nbk_fof_link(None, 4, None, None, -1, None, None, 5, 1, box, org, nc, 1.0, None, None, None) == -1 \
        and b"id base" in err()
    assert L.nbk_fof_link(None, 4, None, None, 0, None, None, 5, 1, box, org, nc, -1.0, None, None, None) == -1 \
        and b"linking length" in err()
    assert L.nbk_fof_finalize(None, None, -1, None, None, None, None, None) == -1 and b"out of range" in err()
    assert L.nbk_fof_lower(None, 1 << 32, None, 4, None, None, None, None) == -1 and b"out of range" in err()
    assert L.nbk_fof_root_counts(None, -1, None, None) == -1 and b"out of range" in err()
    assert L.nbk_fof_label_rows(None, 10, None, None, 2, None) == -1 and b"4- or 8-byte" in err()
    assert L.nbk_fof_segment_reduce(7, None, 4, None, 8, None, None, 1, box, None, None, None, 1, None, 1, None, None,
                                    None) == -1 and b"bad op" in err()
    assert L.nbk_fof_segment_reduce(0, None, 5, None, 8, None, None, 1, box, None, None, None, 1, None, 1, None, None,
                                    None) == -1 and b"column dtype" in err()
    assert L.nbk_fof_segment_reduce(2, None, 4, ctypes.c_void_p(8), 8, None, None, 1, box, None, None, None, 1, None, 1,
                                    None, None, None) == -1 and b"thresholds" in err()


def _cpu_cat(cols, **attrs):
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.lab import ArrayCatalog
    return ArrayCatalog(cols, comm=SelfComm(), **attrs)


def test_fof_host_errors():
    from nbodykit_b200.lab import FOF
    pos = np.random.RandomState(0).uniform(size=(10, 3))
    with pytest.raises(ValueError, match="Position"):
        FOF(_cpu_cat({"X": pos}, BoxSize=1.0), 0.2, 5)
    with pytest.raises(ValueError, match="BoxSize"):
        FOF(_cpu_cat({"Position": pos}), 0.2, 5, absolute=True)
    with pytest.raises(ValueError, match="linking length"):
        FOF(_cpu_cat({"Position": pos}, BoxSize=[1., 1., 1.]), 0.0, 5, absolute=True)


def test_features_and_halos_errors_without_running(monkeypatch):
    """find_features and to_halos check their inputs before any device work"""
    from nbodykit_b200.algorithms.fof import FOF
    monkeypatch.setattr(FOF, "run", lambda self: None)
    pos = np.random.RandomState(0).uniform(size=(10, 3))
    fof = FOF(_cpu_cat({"Position": pos}, BoxSize=[1., 1., 1.]), 0.2, 5)
    assert fof.attrs == dict(linking_length=0.2, nmin=5, absolute=False, periodic=True, domain_factor=1)
    assert abs(fof._linking_length - 0.2 * (1. / 10) ** (1 / 3.)) < 1e-15
    with pytest.raises(ValueError, match="Velocity"):
        fof.find_features()
    with pytest.raises(NotImplementedError, match="halotools"):
        fof.to_halos(1e12, None, 0.5)


def test_cells_per_axis_cap():
    """2^21 cells of side b / sqrt(3) on an axis are accepted, 2^21 + 1 are not, nor 2^21 on all three axes (a 63-bit
    key); one cell at least, and the ceil boundary a relative 1e-11 either side"""
    from nbodykit_b200.algorithms.fof import _cells
    b = 1.
    per_cell = b / (np.sqrt(3) * (1 + 1e-9))
    assert _cells([((1 << 21) - 0.5) * per_cell, 1., 1.], b) == [1 << 21, 2, 2]
    assert _cells([1., 1., ((1 << 21) - 0.5) * per_cell], b) == [2, 2, 1 << 21]
    with pytest.raises(ValueError, match="63-bit"):
        _cells([((1 << 21) + 0.5) * per_cell, 1., 1.], b)
    with pytest.raises(ValueError, match="63-bit"):
        _cells([((1 << 21) - 0.5) * per_cell] * 3, b)
    assert _cells([((1 << 20) + 0.5) * per_cell] * 3, b) == [(1 << 20) + 1] * 3
    assert _cells([1e-300, 1e-3, 0.5], b) == [1, 1, 1]
    L, n = 20., 13
    b0 = L * np.sqrt(3) * (1 + 1e-9) / n
    assert _cells([L] * 3, b0 * (1 - 1e-11)) == [n + 1] * 3
    assert _cells([L] * 3, b0 * (1 + 1e-11)) == [n] * 3


def test_fof_is_exported():
    import nbodykit_b200.algorithms as alg
    import nbodykit_b200.lab as lab
    assert "FOF" in alg.__all__ and lab.FOF is alg.FOF


def test_oracle_on_hand_made_cases():
    # a chain across the periodic face, an isolated pair, singletons
    pos = np.array([[9.9, 5, 5], [0.2, 5, 5], [0.6, 5, 5], [3, 3, 3], [3, 3, 3.4], [7, 7, 7], [1, 8, 8]])
    lab = fo.fof_labels(pos, 0.5, 1, [10.] * 3)
    np.testing.assert_array_equal(lab, [1, 1, 1, 2, 2, 0, 0])
    lab0 = fo.fof_labels(pos, 0.5, 0, [10.] * 3)
    np.testing.assert_array_equal(lab0, [1, 1, 1, 2, 2, 3, 4])          # equal sizes: by smallest member
    np.testing.assert_array_equal(fo.fof_labels(pos, 0.5, 0, None), [3, 1, 1, 2, 2, 4, 5])
    f = fo.features(lab, pos, np.ones_like(pos), [10.] * 3)
    np.testing.assert_allclose(f["CMPosition"][1], [(9.9 + 10.2 + 10.6) / 3 - 10, 5, 5])
    assert f["Length"].tolist() == [0, 3, 2]


def test_oracle_refuses_pairs_at_the_threshold():
    pos = np.array([[0., 0., 0.], [0.5, 0., 0.]])
    with pytest.raises(AssertionError):
        fo.friend_pairs(pos, 0.5, [10.] * 3)
