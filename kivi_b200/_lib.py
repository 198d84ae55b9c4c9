"""ctypes loader for libkivi_b200.so (the C-ABI declared in include/kivi_b200.h).

There is NO fallback: if the CUDA library is missing or a tensor is not on a CUDA device the
call raises.  Nothing in this package imports oracle/.
"""
from __future__ import annotations

import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("KIVI_B200_LIB") or os.path.join(_HERE, "csrc", "libkivi_b200.so")   # override: tuning builds
_LIB = None

_i32, _i64, _vp = ctypes.c_int, ctypes.c_int64, ctypes.c_void_p

_SIGNATURES = {
    "kivi_version": (ctypes.c_int, []),
    "kivi_error_string": (ctypes.c_char_p, [_i32]),
    "kivi_launch_count": (ctypes.c_uint64, []),
    "kivi_pack_lastdim_f16": (_i32, [_vp, _i64, _i64, _i32, _i32, _vp, _vp, _vp, _vp]),
    "kivi_unpack_dequant_lastdim_f16": (_i32, [_vp, _vp, _vp, _i64, _i64, _i32, _i32, _vp, _vp]),
    "kivi_bgemv_outer_f16": (_i32, [_vp, _i64, _vp, _i64, _i64, _vp, _vp, _i64, _i64, _vp,
                                    _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "kivi_gemv_inner_f16": (_i32, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i64, _vp]),
}


class KiviError(RuntimeError):
    def __init__(self, fn: str, code: int, msg: str):
        super().__init__(f"{fn} failed: {msg} (code {code})")
        self.code = code


def lib() -> ctypes.CDLL:
    """Load libkivi_b200.so; raise loudly if it has not been built (python -m kivi_b200.build)."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(SO_PATH):
            raise RuntimeError(
                f"kivi_b200: CUDA library {SO_PATH} is missing. Build it with `python -m kivi_b200.build` "
                "(nvcc, sm_90a). There is no CPU or PyTorch fallback for this package.")
        L = ctypes.CDLL(SO_PATH)
        for name, (res, args) in _SIGNATURES.items():
            if hasattr(L, name):
                fn = getattr(L, name)
                fn.restype, fn.argtypes = res, args
        _LIB = L
    return _LIB


def bind(name: str, restype, argtypes):
    """Declare the signature of an additional exported symbol (used by the cache/decode modules)."""
    fn = getattr(lib(), name)
    fn.restype, fn.argtypes = restype, argtypes
    return fn


def check(code: int, fn: str):
    if code != 0:
        raise KiviError(fn, code, lib().kivi_error_string(code).decode())


def stream_ptr(device=None) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def require_cuda(*tensors: torch.Tensor):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("kivi_b200 operates on CUDA tensors only (no CPU fallback); got a tensor on "
                               f"{t.device}")


def launch_count() -> int:
    return int(lib().kivi_launch_count())
