"""LoRA adapter for the QuantLinear epilogue hook (`forward()` calls `adapter.apply(x=x, out=out)`).

Same interface and arithmetic as the reference's `Lora` (gptqmodel/adapter/adapter.py:116-260):
``out += (x @ lora_A) @ lora_B`` with ``lora_A [in_features, r]`` and ``lora_B [r, out_features]`` (the transposes of
PEFT's ``<module>.lora_A.weight [r, K]`` / ``<module>.lora_B.weight [N, r]``), matrices moved to the activations' dtype
and device on first use.  The two skinny GEMMs are plain dense library GEMMs (cuBLAS through torch): they are not the
quantised hot path.  `post_init(weight_key, device, lora_A=None, lora_B=None)` takes preloaded tensors or finds them by
key suffix in ``<path>/adapter_model.safetensors`` (or `path` itself if it is a .safetensors file).
"""
from __future__ import annotations

import os
from typing import List, Optional

import torch

ADAPTER_FILE = "adapter_model.safetensors"


class Lora:
    def __init__(self, rank: Optional[int] = None, path: Optional[str] = None, lora_A: Optional[torch.Tensor] = None,
                 lora_B: Optional[torch.Tensor] = None):
        self.rank, self.path = rank, path
        self.lora_A, self.lora_B = lora_A, lora_B

    @classmethod
    def name(cls) -> str:
        return "lora"

    @classmethod
    def parameter_keys(cls) -> List[str]:
        return ["lora_A", "lora_B"]

    def apply(self, x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
        if self.lora_A is None or self.lora_B is None:
            raise RuntimeError("Lora.apply() before post_init(): lora_A / lora_B are not loaded")
        if x.dtype != self.lora_A.dtype or x.device != self.lora_A.device:
            self.lora_A = self.lora_A.to(device=x.device, dtype=x.dtype)
            self.lora_B = self.lora_B.to(device=x.device, dtype=x.dtype)
        x2 = x.reshape(-1, x.shape[-1])
        delta = (x2 @ self.lora_A) @ self.lora_B
        return out.add_(delta.view(out.shape))

    def post_init(self, weight_key: str, device, lora_A: Optional[torch.Tensor] = None,
                  lora_B: Optional[torch.Tensor] = None):
        if lora_A is None or lora_B is None:
            if self.lora_A is not None and self.lora_B is not None:
                lora_A, lora_B = self.lora_A, self.lora_B
            elif self.path is not None:
                lora_A, lora_B = self._load(weight_key)
            else:
                raise ValueError("Lora.post_init(): no tensors given and no `path` to load them from")
        if lora_A.shape[1] != lora_B.shape[0]:
            raise ValueError(f"Lora: lora_A {tuple(lora_A.shape)} and lora_B {tuple(lora_B.shape)} do not share a rank")
        if self.rank is not None and self.rank != lora_A.shape[1]:
            raise ValueError(f"Lora: `rank` must match the loaded matrices, expected {self.rank}, got {lora_A.shape[1]}")
        self.rank = lora_A.shape[1]
        keep = lambda t: t.to(device=device, dtype=torch.float32 if t.dtype == torch.float64 else t.dtype).contiguous()  # noqa: E731
        self.lora_A, self.lora_B = keep(lora_A), keep(lora_B)

    def _load(self, weight_key: str):
        from safetensors import safe_open

        fn = self.path if self.path.endswith(".safetensors") else os.path.join(self.path, ADAPTER_FILE)
        key = weight_key.lower()
        a = b = None
        with safe_open(fn, framework="pt") as f:
            for k in f.keys():
                kl = k.lower()
                if kl.endswith(f"{key}.lora_a.weight"):
                    a = f.get_tensor(k).T              # PEFT stores [r, K]
                elif kl.endswith(f"{key}.lora_b.weight"):
                    b = f.get_tensor(k).T.contiguous()  # PEFT stores [N, r]
        if a is None or b is None:
            raise KeyError(f"Lora: `{weight_key}.lora_A.weight` / `.lora_B.weight` not found in {fn}")
        return a, b

    def to_dict(self):
        return {"name": self.name(), "path": self.path, "rank": self.rank}
