"""Loader of the nvcc-built CUDA library.  There is no other backend: if the extension is missing
this raises instead of falling back to anything."""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build
from ._binding import bind

_cdll = None


class ExtensionMissing(RuntimeError):
    pass


def library_path() -> str:
    return _build.OUT


def load() -> C.CDLL:
    global _cdll
    if _cdll is None:
        path = library_path()
        if not os.path.exists(path):
            raise ExtensionMissing(
                f"{path} not built: run `python -m distributed_plonk_b200.build` (nvcc, sm_90a). "
                "distributed_plonk_b200 has no CPU or pure-Python path.")
        _cdll = bind(C.CDLL(path))
    return _cdll
