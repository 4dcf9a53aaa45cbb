"""gptqmodel_b200 — H100-native (sm_90a) GPTQ W4A16/W8A16 QuantLinear hot path.

Public API:
    B200QuantLinear   drop-in QuantLinear (reference contract: gptqmodel/nn_modules/qlinear)
    B200AwqQuantLinear / awq_gemm_to_gptq   AWQ GEMM-format front-end onto the same kernels
    lib / check       the raw C-ABI (include/b2q.h) through ctypes
"""
from ._lib import ABI_VERSION, B2QError, LIB_PATH, SYMBOLS, check, lib  # noqa: F401
from .qlinear import B200QuantLinear, SiblingGroup, fuse_siblings  # noqa: F401
from .adapter import Lora  # noqa: F401
from .awq import B200AwqQuantLinear, awq_gemm_to_gptq  # noqa: F401

__all__ = ["B200QuantLinear", "B200AwqQuantLinear", "awq_gemm_to_gptq", "Lora", "fuse_siblings", "SiblingGroup", "lib", "check", "B2QError", "LIB_PATH", "SYMBOLS", "ABI_VERSION"]
