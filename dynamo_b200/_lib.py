"""Locates and loads the in-tree native libraries.  Fails loudly: there is no CPU fallback."""
from __future__ import annotations

import ctypes as C
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
KERNELS_SO = os.path.join(_PKG, "libkvbm_kernels.so")
PHYSICAL_SO = os.path.join(_PKG, "libkvbm_physical.so")


class NativeLibraryMissing(RuntimeError):
    pass


_cache: dict[str, C.CDLL] = {}


def load(path: str) -> C.CDLL:
    lib = _cache.get(path)
    if lib is None:
        if not os.path.exists(path):
            raise NativeLibraryMissing(
                f"{path} is not built. Run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). dynamo_b200 has no CPU fallback for the KV transfer path.")
        lib = C.CDLL(path, mode=C.RTLD_GLOBAL)
        _cache[path] = lib
    return lib
