"""Target for one `ncu --set full --profile-from-start off` capture of the HEAD decode / act-order staging kernels:
decode_kernel (4096x4096 plain and act-order, 14336x4096 act-order), decode2_kernel (4096x14336), permute_rows_kernel
(M = 2048 act-order prefill).  Weights rotate over 8 distinct layers per shape so every captured launch reads HBM-cold."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gptqmodel_b200 import B200QuantLinear  # noqa: E402
from helpers import random_layer  # noqa: E402


def build(K, N, act, n=6):
    mods = []
    for i in range(n):
        L = random_layer(K, N, bits=4, group_size=128, sym=True, seed=K + N + i, device="cuda")
        if act:
            perm = torch.randperm(K, generator=torch.Generator().manual_seed(i))
            L["g_idx"] = (torch.arange(K, dtype=torch.int32) // 128)[perm].cuda()
        mods.append(B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4, 128,
                                                            desc_act=act))
    return mods


cases = [("o_proj plain", build(4096, 4096, False)), ("gate|up-size plain", build(4096, 14336, False)),
         ("o_proj act-order", build(4096, 4096, True)), ("down_proj act-order", build(14336, 4096, True))]
xs = {K: (torch.randn(1, K, device="cuda") * 0.5).half() for K in (4096, 14336)}
xp = (torch.randn(2048, 4096, device="cuda") * 0.5).half()
for _ in range(2):
    for name, mods in cases:
        for m in mods[:-1]:
            m(xs[m.in_features])
    cases[2][1][0](xp)
torch.cuda.synchronize()
torch.cuda.profiler.start()
for name, mods in cases:
    mods[-1](xs[mods[-1].in_features])   # the layer not touched during warm-up: HBM-cold weights
cases[2][1][-1](xp)                      # act-order prefill: permute_rows_kernel + gemm_kernel
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print("captured", [c[0] for c in cases], "+ act-order prefill")
