"""embree_b200 -- H100-native ray tracing kernels behind the Embree 4 C API.

The product is the C-ABI shared library embree_b200/csrc/libembree4_b200.so (hand-written sm_90a CUDA +
the C++ host shim); this package only locates/loads it for the Python tests and bench.py.  There is no CPU or
PyTorch fallback: if the library has not been built (python __graft_entry__.py / make -C embree_b200/csrc),
`load()` raises.
"""
import os

from .rtc import RTCLib  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
# EMBREE_B200_LIB: A/B measurements of alternative BUILDS of this same library (scripts/ab.py); never a fallback
LIB_PATH = os.environ.get("EMBREE_B200_LIB") or os.path.join(_HERE, "csrc", "libembree4_b200.so")
_lib = None


def load():
    """Load (once) and return the product library as an RTCLib binding."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a).  embree_b200 has no CPU fallback.")
        _lib = RTCLib(LIB_PATH)
        if not _lib.is_b200:
            raise RuntimeError(f"{LIB_PATH} does not export the rtcb200* entry points")
    return _lib
