"""kajiya_b200 — H100-native (sm_90a CUDA) implementation of kajiya's ReSTIR-GI hot path.

The package is a thin host-side mirror of the reference's renderer API over the C-ABI shared
library `kajiya_b200/csrc/libkjb.so` (hand-written CUDA kernels + the C++ frame driver).
There is NO CPU fallback: importing `lib()` without the built CUDA library, or creating a
context without a CUDA device, raises.
"""
import os
from ._abi import KjbLib, KjbError, Image, WorldDesc, WorldFrame, MeshDesc, MeshMaterial, TextureDesc, FMT, FMT_NAME, FMT_NUMPY
from .world import World
from . import scenes

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libkjb.so")
_lib = None


def lib():
    """The CUDA implementation.  Fails loudly when the extension has not been built (python __graft_entry__.py build)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise KjbError(f"CUDA extension missing: {LIB_PATH} (run `python -c 'import __graft_entry__ as g; g.build()'`). "
                           "kajiya_b200 has no CPU fallback.")
        _lib = KjbLib(LIB_PATH)
        if _lib.backend != "cuda-sm90a":
            raise KjbError(f"unexpected backend {_lib.backend!r} behind {LIB_PATH}")
    return _lib


FAST_LIB_PATH = os.path.join(_HERE, "csrc", "libkjb_fast.so")
_fast = None


def lib_fast():
    """The same kernels compiled with -DKJB_FAST -use_fast_math (MUFU transcendentals, approximate division / sqrt, FMA contraction): NOT
    bit-compatible with the oracle, never returned by lib().  Exists so that the cost of the exact numeric contract is a measured number
    (bench.py `fast_math`, tests/test_gpu_fast.py)."""
    global _fast
    if _fast is None:
        if not os.path.exists(FAST_LIB_PATH):
            raise KjbError(f"fast-math build missing: {FAST_LIB_PATH}")
        _fast = KjbLib(FAST_LIB_PATH)
        if _fast.backend != "cuda-sm90a-fast":
            raise KjbError(f"unexpected backend {_fast.backend!r} behind {FAST_LIB_PATH}")
    return _fast
