"""ctypes binding of embree_b200/csrc/libpathstream_b200.so: the wavefront path-tracer driver kernels (primary rays,
bounce, shade) that turn BASELINE configs[4] into a stream of batched rtcIntersect1 / rtcOccluded1 calls.  All pointers
are device memory; the caller owns the buffers (PyTorch tensors in bench.py and the tests)."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libpathstream_b200.so")
_lib = None


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: build it with `make -C embree_b200/csrc` (nvcc, sm_90a); there is no fallback")
        d = C.CDLL(LIB_PATH)
        d.pts200_primary.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_ulonglong, C.c_uint, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
        d.pts200_bounce.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p]
        d.pts200_shade.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p]
        _lib = d
    return _lib
