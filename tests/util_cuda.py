"""libcudart through ctypes, for tests that reach device memory without going through the library: an index's arrays
(Index.layout()) copied device-to-device for replicas or device-to-host to compare them with a CPU computation, and a
batch's result rows (Batch.device_results()) read back or poisoned before a rerun."""
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
        _rt.cudaMemset.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t]
    return _rt


def download(dev_ptr, nbytes, dtype):
    """Bytes [dev_ptr, dev_ptr + nbytes) of device memory as a host array of `dtype`."""
    out = np.empty(nbytes, dtype=np.uint8)
    assert cudart().cudaMemcpy(out.ctypes.data, dev_ptr, nbytes, D2H) == 0
    return out.view(dtype)


def memset(dev_ptr, value, nbytes):
    """Every byte of [dev_ptr, dev_ptr + nbytes) set to `value`.  On the legacy default stream, which does not wait for
    non-blocking streams (the library's): finish their work first, and call device_synchronize() before they read."""
    assert cudart().cudaMemset(dev_ptr, value, nbytes) == 0


def device_synchronize():
    assert cudart().cudaDeviceSynchronize() == 0


def free_bytes():
    free, total = ctypes.c_size_t(), ctypes.c_size_t()
    assert cudart().cudaMemGetInfo(ctypes.byref(free), ctypes.byref(total)) == 0
    return free.value


def sm_count(device=0):
    """Streaming multiprocessors of `device` (cudaDevAttrMultiProcessorCount)."""
    v = ctypes.c_int(0)
    assert cudart().cudaDeviceGetAttribute(ctypes.byref(v), 16, device) == 0
    return v.value
