"""Phase timeline of the decode kernel (debug stamps), inside a CUDA graph of back-to-back launches."""
import os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import gptqmodel_b200 as g
from gptqmodel_b200 import B200QuantLinear
from helpers import random_layer
K, N = int(sys.argv[1]), int(sys.argv[2])
mods = []
for c in range(12):
    L = random_layer(K, N, seed=c, device="cuda")
    mods.append(B200QuantLinear.from_checkpoint_tensors(L["qweight"], L["qzeros"], L["scales"], L["g_idx"], 4, 128, device="cuda"))
x = (torch.randn(1, K, device="cuda") * 0.5).to(torch.float16)
traces = [torch.zeros(160 * 16, dtype=torch.int64, device="cuda") for _ in mods]
def fn():
    for m, tr in zip(mods, traces):
        g.lib.b2q_debug_set_trace(tr.data_ptr())
        m(x)
    g.lib.b2q_debug_set_trace(None)
s = torch.cuda.Stream(); s.wait_stream(torch.cuda.current_stream())
with torch.cuda.stream(s): fn()
torch.cuda.current_stream().wait_stream(s)
gr = torch.cuda.CUDAGraph()
with torch.cuda.graph(gr): fn()
for _ in range(3): gr.replay()
torch.cuda.synchronize()
T = torch.stack(traces).cpu().reshape(len(mods), 160, 16).double()
base = T[6][:, 0].min()
for li in (6, 7):
    t = T[li] - base
    used = t[:, 0] > -1e8
    names = ["start", "issued", "gdc_wait", "staged"] + [f"t{i//2}{'b' if i%2 else 'a'}" for i in range(10)] + ["?", "end"]
    if os.environ.get("B2Q_DECODE_V2") == "1":  # b2q_decode2.cu stamps: no per-tile epilogues
        names[4], names[5] = "loop_done", "cta_reduced"
    print(f"layer {li}:  (ns relative to layer 6's first CTA start; min / median / max over CTAs)")
    for sl in range(16):
        col = t[:, sl][T[li][:, sl] > 0]
        if col.numel():
            print(f"   {names[sl]:9s} {col.min().item():9.0f} {col.median().item():9.0f} {col.max().item():9.0f}   n={col.numel()}")
