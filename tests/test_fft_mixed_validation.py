"""Argument validation of the mixed-radix FFT entry points: every rejected call returns -1 with a message before any
CUDA call, so these run on a host without a GPU."""
from nbodykit_b200 import _lib


def test_r2c_mixed_rejects_unsupported_sizes():
    L = _lib.lib()
    for nmesh in ([11, 12, 12], [12, 22, 12], [12, 12, 13]):          # prime factors 11 and 13
        assert L.nbk_r2c_mixed(None, None, 8, _lib.iarr(nmesh), 1.0, None) == -1
        msg = L.nbk_last_error()
        assert b"2, 3, 5 and 7" in msg and b"4096" in msg
    for nmesh in ([4608, 12, 12], [12, 4116, 12], [12, 12, 8232], [12, 12, 4375], [1, 12, 12]):   # outside the limits
        assert L.nbk_r2c_mixed(None, None, 8, _lib.iarr(nmesh), 1.0, None) == -1
        assert b"unsupported" in L.nbk_last_error()
    assert L.nbk_c2r_mixed(None, None, 4, _lib.iarr([11, 12, 12]), None, None) == -1
    assert b"unsupported" in L.nbk_last_error()


def test_mixed_entry_points_reject_bad_dtype():
    L = _lib.lib()
    assert L.nbk_r2c_mixed(None, None, 3, _lib.iarr([12, 12, 12]), 1.0, None) == -1 and b"dtype" in L.nbk_last_error()
    assert L.nbk_c2r_mixed(None, None, 16, _lib.iarr([12, 12, 12]), None, None) == -1 and b"dtype" in L.nbk_last_error()
    assert L.nbk_fft_lines_mixed(None, None, 3, 12, 1, 1, 1, 12, 0, 1.0, None) == -1 and b"dtype" in L.nbk_last_error()
    assert L.nbk_fft_z_mixed(None, None, 3, 4, 12, 0, 1.0, None) == -1 and b"dtype" in L.nbk_last_error()


def test_line_and_z_passes_reject_length_13():
    L = _lib.lib()
    assert L.nbk_fft_lines_mixed(None, None, 8, 13, 1, 1, 1, 13, 0, 1.0, None) == -1
    assert b"line length 13" in L.nbk_last_error()
    assert L.nbk_fft_z_mixed(None, None, 8, 4, 13, 0, 1.0, None) == -1
    assert b"Nz = 13" in L.nbk_last_error()
    # the limits: 4096-point lines, z rows of 8192 (even) / 4095 (odd)
    assert L.nbk_fft_lines_mixed(None, None, 4, 4116, 1, 1, 1, 4116, 0, 1.0, None) == -1
    assert L.nbk_fft_lines_mixed(None, None, 4, 1, 1, 1, 1, 1, 0, 1.0, None) == -1
    assert L.nbk_fft_z_mixed(None, None, 4, 4, 8232, 0, 1.0, None) == -1
    assert L.nbk_fft_z_mixed(None, None, 4, 4, 4375, 1, 1.0, None) == -1


def test_empty_work_needs_no_gpu():
    """valid sizes with nothing to transform return 0 without a launch"""
    L = _lib.lib()
    assert L.nbk_fft_lines_mixed(None, None, 8, 96, 1, 0, 1, 96, 0, 1.0, None) == 0
    assert L.nbk_fft_z_mixed(None, None, 8, 0, 100, 0, 1.0, None) == 0


def test_version_bumped_for_the_mixed_path():
    assert _lib.lib().nbk_version() >= 101


def test_particle_mesh_flags_power_of_two_sides():
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.pmesh.pm import ParticleMesh
    assert ParticleMesh(BoxSize=1.0, Nmesh=64, dtype='f4', comm=SelfComm()).pow2
    assert not ParticleMesh(BoxSize=1.0, Nmesh=96, dtype='f4', comm=SelfComm()).pow2
    assert not ParticleMesh(BoxSize=1.0, Nmesh=[64, 64, 45], dtype='f8', comm=SelfComm()).pow2
