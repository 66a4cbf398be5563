"""Loader of the native extension.

The CUDA path must never silently degrade: if the shared object is missing it is built
in-tree (nvcc, sm_90a); if that is impossible an ImportError with the build log is raised.
"""
from __future__ import annotations

import importlib
import threading

_lock = threading.Lock()
_mod = None


def C():
    """Return the pybind11 module ``uccl_b200._C`` (building it on first use if needed)."""
    global _mod
    if _mod is not None:
        return _mod
    with _lock:
        if _mod is not None:
            return _mod
        try:
            _mod = importlib.import_module("uccl_b200._C")
        except ImportError:
            from . import _build

            _build.build()
            _mod = importlib.import_module("uccl_b200._C")
        return _mod


def is_built() -> bool:
    from . import _build

    return _build.module_path().exists()


def module_path() -> str:
    """Filesystem path of the loaded extension (exports the C symbols torch's pluggable allocator needs)."""
    return C().__file__
