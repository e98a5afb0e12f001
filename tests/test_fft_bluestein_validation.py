"""Argument validation of the Bluestein FFT entry points and the per-axis choice of ParticleMesh: every rejected call
returns -1 with a message before any CUDA call, so these run on a host without a GPU."""
from nbodykit_b200 import _lib


def test_bluestein_entry_points_reject_bad_dtype():
    L = _lib.lib()
    assert L.nbk_fft_lines_bluestein(None, None, 3, 11, 1, 1, 1, 11, 0, 1.0, None) == -1
    assert b"dtype" in L.nbk_last_error()
    assert L.nbk_fft_z_bluestein(None, None, 16, 4, 13, 0, 1.0, None) == -1
    assert b"dtype" in L.nbk_last_error()


def test_bluestein_line_pass_rejects_lengths_outside_2_to_4096():
    L = _lib.lib()
    for n in (1, 4097, 4116):
        assert L.nbk_fft_lines_bluestein(None, None, 8, n, 1, 1, 1, n, 0, 1.0, None) == -1
        msg = L.nbk_last_error()
        assert (b"line length %d" % n) in msg and b"2 .. 4096" in msg


def test_bluestein_z_pass_rejects_lengths_outside_the_limits():
    L = _lib.lib()
    for nz in (8194, 4097, 1):
        assert L.nbk_fft_z_bluestein(None, None, 4, 4, nz, 0, 1.0, None) == -1
        msg = L.nbk_last_error()
        assert (b"Nz = %d" % nz) in msg and b"8192" in msg and b"4095" in msg


def test_bluestein_empty_work_needs_no_gpu():
    """valid lengths with nothing to transform return 0 without a launch"""
    L = _lib.lib()
    for n in (11, 13, 4093):
        assert L.nbk_fft_lines_bluestein(None, None, 8, n, 1, 0, 1, n, 0, 1.0, None) == 0
        assert L.nbk_fft_lines_bluestein(None, None, 4, n, 1, 1, 0, n, 1, 1.0, None) == 0
        assert L.nbk_fft_z_bluestein(None, None, 8, 0, n, 0, 1.0, None) == 0


def test_version_bumped_for_the_bluestein_path():
    assert _lib.lib().nbk_version() >= 103


def test_particle_mesh_flags_sides_with_prime_factors_above_7():
    from nbodykit_b200.comm import SelfComm
    from nbodykit_b200.pmesh.pm import ParticleMesh

    def pm(N):
        return ParticleMesh(BoxSize=1.0, Nmesh=N, dtype='f4', comm=SelfComm())
    assert pm([11, 12, 13]).bluestein == (True, False, True)
    assert pm([176, 96, 96]).bluestein == (True, False, False)
    assert pm(96).bluestein == (False, False, False) and not pm(96).pow2
    assert pm(64).bluestein == (False, False, False) and pm(64).pow2
    assert pm([44, 44, 37]).bluestein == (True, True, True)
