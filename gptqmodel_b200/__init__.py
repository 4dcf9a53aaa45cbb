"""gptqmodel_b200 — H100-native (sm_90a) GPTQ W4A16/W8A16 QuantLinear hot path.

Public API:
    B200QuantLinear   drop-in QuantLinear (reference contract: gptqmodel/nn_modules/qlinear)
    B200AwqQuantLinear / awq_gemm_to_gptq   AWQ GEMM-format front-end onto the same kernels
    B200QqqQuantLinear  QQQ (W4A8) checkpoints on the int8 tensor cores
    B200Fp8QuantLinear  FP8 (e4m3fn, W8A16) checkpoints on the 8-bit tiers
    B200BlockFp8Linear  HF / DeepSeek-native block-FP8 (W8A8) checkpoints on the e4m3 tensor cores
    B200ChannelFp8Linear  per-channel / per-tensor FP8 (W8A8: compressed-tensors FP8 / FP8_DYNAMIC, fbgemm_fp8)
    B200ChannelInt8Linear per-channel / per-tensor INT8 (W8A8: compressed-tensors int-quantized) on the s8 tensor cores
    B200W4Fp8Linear   W4AFP8 (compressed-tensors pack-quantized 4-bit group-128 weights, per-token e4m3 activations)
    MoEExperts / B200ChannelW8A8Experts  MoE expert blocks; the latter runs W8A8 channel experts on grouped kernels
    lib / check       the raw C-ABI (include/b2q.h) through ctypes
"""
from ._lib import ABI_VERSION, B2QError, LIB_PATH, SYMBOLS, check, lib  # noqa: F401
from .qlinear import B200QuantLinear, SiblingGroup, fuse_siblings  # noqa: F401
from .adapter import Lora  # noqa: F401
from .awq import B200AwqQuantLinear, awq_gemm_to_gptq  # noqa: F401
from .qqq import B200QqqQuantLinear  # noqa: F401
from .fp8 import B200Fp8QuantLinear  # noqa: F401
from .fp8_block import B200BlockFp8Linear  # noqa: F401
from .fp8_channel import B200ChannelFp8Linear  # noqa: F401
from .int8_channel import B200ChannelInt8Linear  # noqa: F401
from .w4afp8 import B200W4Fp8Linear  # noqa: F401
from .moe import B200ChannelW8A8Experts, MoEExperts, route_grouped_sigmoid, route_softmax_topk  # noqa: F401

__all__ = ["B200QuantLinear", "B200AwqQuantLinear", "B200QqqQuantLinear", "B200Fp8QuantLinear", "B200BlockFp8Linear", "B200ChannelFp8Linear", "B200ChannelInt8Linear", "B200W4Fp8Linear", "B200ChannelW8A8Experts", "MoEExperts", "awq_gemm_to_gptq", "Lora", "fuse_siblings", "SiblingGroup", "lib", "check", "B2QError", "LIB_PATH", "SYMBOLS", "ABI_VERSION"]
