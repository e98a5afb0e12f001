"""
Small ctypes / torch helpers shared by the virtual-rank GPU tests (tests/test_gpu_slab_fft.py,
tests/test_gpu_slab_route.py).  Importing this module needs neither a GPU nor the built library.
"""
import ctypes

import numpy as np


def nbk():
    """the nbodykit_b200._lib module (the ctypes binding), imported on first use"""
    from nbodykit_b200 import _lib
    return _lib


def ptr(t):
    """device pointer of a tensor as the C ABI takes it (None stays NULL)"""
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def code(dt):
    """NBK_F4 / NBK_F8 of a float32 / float64 dtype ('f4', np.float32, np.dtype('f8'), ...)"""
    return 4 if np.dtype(dt) == np.float32 else 8


def dev(a):
    """a host array as a contiguous tensor on the current device"""
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    """a device tensor as numpy, after the device has finished the work queued on it"""
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy()
