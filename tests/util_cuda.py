"""libcudart through ctypes, for tests that copy an index's device arrays (Index.layout()) without going through the
library: device-to-device for replicas, device-to-host to compare the arrays with a CPU computation."""
import ctypes

import numpy as np

H2D, D2H, D2D = 1, 2, 3  # cudaMemcpyKind

_rt = None


def cudart():
    global _rt
    if _rt is None:
        for name in ("libcudart.so", "libcudart.so.12", "/usr/local/cuda/lib64/libcudart.so"):
            try:
                _rt = ctypes.CDLL(name)
                break
            except OSError:
                pass
        assert _rt is not None, "libcudart not found"
        _rt.cudaMemcpy.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int]
    return _rt


def download(dev_ptr, nbytes, dtype):
    """Bytes [dev_ptr, dev_ptr + nbytes) of device memory as a host array of `dtype`."""
    out = np.empty(nbytes, dtype=np.uint8)
    assert cudart().cudaMemcpy(out.ctypes.data, dev_ptr, nbytes, D2H) == 0
    return out.view(dtype)
