"""Loader for the in-tree sm_90a kernel library.

Policy: on a machine with a CUDA device the native library is *required* — any op that receives a CUDA
tensor raises if it cannot be loaded (no silent PyTorch fallback; set ``PFX_ALLOW_FALLBACK=1`` to opt in
for debugging).  On CPU-only machines the pure-PyTorch reference implementations in ``functional.py`` run.
"""
from __future__ import annotations

import importlib.machinery
import importlib.util
import os
from typing import Optional

_lib = None
_load_error: Optional[BaseException] = None
_tried = False


def load(build_if_missing: bool = False):
    global _lib, _load_error, _tried
    if _lib is not None:
        return _lib
    if _tried and not build_if_missing:
        return None
    _tried = True
    try:
        import torch  # noqa: F401  (libtorch symbols must be loaded first)

        from . import build as _build

        path = _build.lib_path()
        if build_if_missing and not _build.is_fresh():
            path = _build.build(verbose=False)
        if not path.exists():
            raise FileNotFoundError(f"{path} not built; run python -m paddlefleetx_b200.ops.build")
        loader = importlib.machinery.ExtensionFileLoader(_build.MODULE_NAME, str(path))
        spec = importlib.util.spec_from_file_location(_build.MODULE_NAME, str(path), loader=loader)
        mod = importlib.util.module_from_spec(spec)
        loader.exec_module(mod)
        _lib = mod
        _load_error = None
    except BaseException as e:  # noqa: BLE001
        _load_error = e
        _lib = None
    return _lib


def available() -> bool:
    return load() is not None


def allow_fallback() -> bool:
    return os.environ.get("PFX_ALLOW_FALLBACK", "0") == "1"


def require():
    lib = load()
    if lib is None:
        raise RuntimeError(
            "paddlefleetx_b200 native kernel library is not available on this CUDA machine "
            f"({_load_error!r}). Build it with `python -m paddlefleetx_b200.ops.build`.")
    return lib


def use_native(*tensors) -> bool:
    """True when the op should run the hand-written CUDA path."""
    import torch

    if not all(t.is_cuda for t in tensors if isinstance(t, torch.Tensor)):
        return False
    if load() is None:
        if allow_fallback():
            return False
        require()
    return True
