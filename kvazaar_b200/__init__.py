"""kvazaar_b200 -- H100 (sm_90a) "cuda" strategy kernels for Kvazaar's per-CTU hot path.

The product is the C-ABI shared library ``libkvzcuda.so`` (include/kvz_cuda.h); this package is the thin
Python plumbing used by the tests and bench.py: it loads the library with ctypes and passes torch CUDA
tensors (device memory + streams are torch's job here, nothing else).  There is NO CPU fallback: importing
works without a GPU (so the CPU test-suite can check the exported symbols), but every compute entry point
raises if the library or a device is missing.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libkvzcuda.so")


class KvzCudaError(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise KvzCudaError(f"{LIB_PATH} is missing: build it with `make lib` (or __graft_entry__.build()); "
                           "there is no CPU fallback")
    lib = C.CDLL(LIB_PATH)
    lib.kvz_cuda_last_error.restype = C.c_char_p
    lib.kvz_cuda_launch_count.restype = C.c_uint64
    lib.kvz_cuda_strategy_fptr.restype = C.c_void_p
    lib.kvz_cuda_strategy_fptr.argtypes = [C.c_char_p, C.c_uint8]
    for n in ("kvz_cuda_malloc", "kvz_cuda_host_alloc"):
        getattr(lib, n).restype = C.c_void_p
        getattr(lib, n).argtypes = [C.c_size_t]
    return lib


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = _load()
    return _lib


from .api import *  # noqa: E402,F401,F403
