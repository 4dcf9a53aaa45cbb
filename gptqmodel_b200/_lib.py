"""ctypes binding of libb2q.so (C-ABI declared in include/b2q.h).

There is NO fallback: if the CUDA library is missing or fails to load, importing this module raises.
"""
from __future__ import annotations

import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb2q.so")

ABI_VERSION = 3

# every symbol include/b2q.h declares: (restype, argtypes)
_vp, _i, _sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
SYMBOLS = {
    "b2q_version": (_i, []),
    "b2q_last_error": (ctypes.c_char_p, []),
    "b2q_packed_bytes": (_sz, [_i, _i, _i]),
    "b2q_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "b2q_mm_workspace_bytes": (_sz, [_i, _i, _i, _i, _i, _i]),
    "b2q_debug_reload_env": (None, []),
    "b2q_prepack": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp]),
    "b2q_mm": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _sz, _vp]),
    "b2q_decode": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "b2q_decode_multi": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "b2q_gemm_multi": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _sz, _vp]),
    "b2q_gemv": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "b2q_gemm": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _sz, _vp]),
    "b2q_allreduce": (_i, [_vp, _i, _i, _i, _i, _vp, _sz, _i, _vp, _vp]),
    "b2q_decode_allreduce": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _sz, _i, _vp, _vp]),
    "b2q_decode_allreduce_flag_bytes": (_sz, []),
    "b2q_debug_set_trace": (None, [_vp]),
    "b2q_debug_decode_plan": (_i, [_i, _i, _i, _i, _i, _i, _vp]),
    "b2q_permute_cols": (_i, [_vp, _vp, _vp, _i, _i, _vp]),
    "b2q_moe_align": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "b2q_moe_gather": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp]),
    "b2q_moe_gate_up": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "b2q_moe_down": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "b2q_moe_combine": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "b2q_moe_decode_gate_up": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "b2q_moe_decode_act": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "b2q_moe_decode_down": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp]),
}


class B2QError(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `python __graft_entry__.py` or `make -C gptqmodel_b200/csrc` "
            "(nvcc -gencode arch=compute_90a,code=sm_90a). There is no CPU/PyTorch fallback."
        )
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    v = lib.b2q_version()
    if v != ABI_VERSION:
        raise ImportError(f"libb2q.so ABI version {v} != expected {ABI_VERSION}; rebuild")
    return lib


lib = _load()


def check(code: int, what: str):
    if code != 0:
        raise B2QError(f"{what} failed ({code}): {lib.b2q_last_error().decode(errors='replace')}")
