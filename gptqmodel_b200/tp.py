"""Tensor-parallel sharding of GPTQ QuantLinear checkpoint tensors + the row-parallel all-reduce.

The reference has no tensor-parallel code; the rules below are the ones it documents for the
engines it delegates to: scales of a row-parallel act-order layer must be replicated on all ranks
(`marlin_repeat_scales_on_all_ranks`, gptqmodel/utils/marlin.py:300-305), K shards must be whole groups
(`marlin_is_k_full` :296-297, TensorParallelPadderConfig quantization/config.py:1184-1188).

  column-parallel (q,k,v,gate,up / expert w1,w3): rank r owns output features [r*N/P, (r+1)*N/P)  -> no comm
  row-parallel    (o_proj, down_proj / expert w2): rank r owns input rows    [r*K/P, (r+1)*K/P)  -> partial sums,
                  ONE all-reduce(sum) of the [M, N] output per layer; bias is added on rank 0 only.

All functions work on checkpoint-layout tensors on any device (they are pure slicing), so the host logic is
testable with the gloo backend on CPU.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.distributed as dist

Layer = Dict[str, object]


def _check(layer: Layer):
    for k in ("qweight", "qzeros", "scales", "g_idx", "bits", "group_size"):
        if k not in layer:
            raise KeyError(f"layer dict misses {k!r}")


def shard_columns(layer: Layer, rank: int, world: int) -> Layer:
    """Column-parallel shard: slice the N axis of qweight / scales / qzeros (qzeros packs 32/bits columns/word)."""
    _check(layer)
    bits = int(layer["bits"])
    pf = 32 // bits
    qweight, qzeros, scales = layer["qweight"], layer["qzeros"], layer["scales"]
    N = qweight.shape[1]
    if N % world != 0 or (N // world) % 32 != 0:
        raise NotImplementedError(f"column shard: N={N} / {world} must be a multiple of 32")
    n0, n1 = rank * N // world, (rank + 1) * N // world
    out = dict(layer)
    out["qweight"] = qweight[:, n0:n1].contiguous()
    out["scales"] = scales[:, n0:n1].contiguous()
    out["qzeros"] = qzeros[:, n0 // pf:n1 // pf].contiguous()
    out["g_idx"] = layer["g_idx"].clone()
    if layer.get("bias") is not None:
        out["bias"] = layer["bias"][n0:n1].contiguous()
    out["N"] = n1 - n0
    return out


def _row_words(k: int, bits: int, planar: bool) -> int:
    """First qweight word row of input feature k (k must start a packing block: 32/bits codes, or 32 for the 3-bit
    stream and the planar layouts)."""
    blk = 32 if (planar or 32 % bits) else 32 // bits
    if k % blk != 0:
        raise NotImplementedError(f"row shard: boundary {k} is not a multiple of the {bits}-bit packing block ({blk})")
    return k * bits // 32


def shard_rows(layer: Layer, rank: int, world: int) -> Layer:
    """Row-parallel shard: slice the K axis (input rows [rank*K/P, (rank+1)*K/P) in CHECKPOINT order).

    Group-contiguous g_idx: K/P must be whole groups; the shard keeps its own rows of the scale / zero tables.
    Act-order g_idx: the shard's rows belong to arbitrary groups, so it keeps the FULL tables (the reference's rule for its
    engines: `marlin_repeat_scales_on_all_ranks`, utils/marlin.py:300-305) and its slice of g_idx still indexes them;
    `B200QuantLinear.post_init` serves such a layer through `layouts.regroup` (out["replicated_tables"] = True)."""
    _check(layer)
    bits = int(layer["bits"])
    planar = bool(layer.get("planar", False))
    qweight, qzeros, scales, g_idx = layer["qweight"], layer["qzeros"], layer["scales"], layer["g_idx"]
    K = g_idx.shape[0]
    gs = int(layer["group_size"])
    gs = gs if gs > 0 else K
    if K % world != 0:
        raise NotImplementedError(f"row shard: K={K} not divisible by {world}")
    k0, k1 = rank * K // world, (rank + 1) * K // world
    out = dict(layer)
    out["qweight"] = qweight[_row_words(k0, bits, planar):_row_words(k1, bits, planar)].contiguous()
    trivial = torch.equal(g_idx.to(torch.int64).cpu(), torch.arange(K) // gs)
    if not trivial:
        out["scales"] = scales.contiguous()
        out["qzeros"] = qzeros.contiguous()
        out["g_idx"] = g_idx[k0:k1].to(torch.int32).contiguous()
        out["replicated_tables"] = True
    elif int(layer["group_size"]) <= 0:
        # one group spans all of K: every rank keeps the single scale row
        out["scales"] = scales[0:1].contiguous()
        out["qzeros"] = qzeros[0:1].contiguous()
        out["g_idx"] = torch.zeros(k1 - k0, dtype=torch.int32, device=g_idx.device)
        out["group_size"] = -1
    else:
        if (k1 - k0) % gs != 0:
            raise NotImplementedError(f"row shard: K/P={k1 - k0} must be a multiple of group_size={gs}")
        g0, g1 = k0 // gs, k1 // gs
        out["scales"] = scales[g0:g1].contiguous()
        out["qzeros"] = qzeros[g0:g1].contiguous()
        out["g_idx"] = (g_idx[k0:k1] - g0).to(torch.int32).contiguous()
    if layer.get("bias") is not None:
        out["bias"] = layer["bias"] if rank == 0 else None  # added once, before the reduce
    out["K"] = k1 - k0
    return out


def shard_moe_expert(w1: Layer, w3: Layer, w2: Layer, rank: int, world: int):
    """One expert of a Mixtral-style MoE block under tensor parallelism (BASELINE configs[4]):
    w1 / w3 (gate / up) column-parallel, w2 (down) row-parallel — every rank keeps a slice of EVERY expert, so the block
    needs one all-reduce of the combined output, exactly like a dense MLP."""
    return shard_columns(w1, rank, world), shard_columns(w3, rank, world), shard_rows(w2, rank, world)


def all_reduce_sum_(t: torch.Tensor, group: Optional[dist.ProcessGroup] = None) -> torch.Tensor:
    """The single collective of a row-parallel QuantLinear: in-place sum over the TP group (NCCL on GPUs)."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
    return t


class P2PAllReduce:
    """One-shot all-reduce(sum) of small 16-bit tensors over NVLink peer memory (`b2q_allreduce`), CUDA-graph safe.

    PyTorch's symmetric-memory rendezvous is used only to allocate the buffer and map the peers' pointers; the
    collective itself is our kernel (gptqmodel_b200/csrc/b2q_allreduce.cu).  Use for the row-parallel QuantLinear
    output at decode time (8-16 KB); large prefill tensors stay on NCCL.
    """

    def __init__(self, device, max_elems: int = 16384, group: Optional[dist.ProcessGroup] = None):
        import ctypes

        import torch.distributed._symmetric_memory as symm_mem

        from ._lib import lib

        self._lib = lib
        group = group if group is not None else dist.group.WORLD
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        if self.world > 8:
            raise NotImplementedError("P2PAllReduce: at most 8 GPUs (one NVLink domain)")
        self.max_elems = (max_elems + 7) // 8 * 8
        self.flag_offset = 2 * self.world * self.max_elems * 2
        nbytes = self.flag_offset + 2 * self.world * 4
        nbytes = (nbytes + 1023) // 1024 * 1024
        self.buf = symm_mem.empty(nbytes // 4, dtype=torch.int32, device=device)
        self.buf.zero_()
        self.hdl = symm_mem.rendezvous(self.buf, group.group_name)
        self._peers = (ctypes.c_void_p * self.world)(*[int(p) for p in self.hdl.buffer_ptrs])
        self.seq = torch.zeros(2, dtype=torch.int32, device=device)  # {call counter, status}
        torch.cuda.synchronize(device)
        dist.barrier(group)  # every rank's buffer is zeroed before anybody pushes into it

    def status(self) -> int:
        """0, or 1 + the rank of a peer whose flag never arrived within the kernel's 2 s bound (host sync; debugging)."""
        return int(self.seq[1].item())

    def __call__(self, t: torch.Tensor) -> torch.Tensor:
        from ._lib import check

        n = t.numel()
        if not t.is_contiguous() or n % 8 != 0 or n > self.max_elems or t.dtype not in (torch.float16, torch.bfloat16):
            raise ValueError("P2PAllReduce: contiguous fp16/bf16 tensor with numel % 8 == 0 and <= max_elems expected")
        check(self._lib.b2q_allreduce(t.data_ptr(), n, 0 if t.dtype == torch.float16 else 1, self.rank, self.world,
                                      self._peers, self.flag_offset, self.max_elems, self.seq.data_ptr(),
                                      torch.cuda.current_stream(t.device).cuda_stream), "b2q_allreduce")
        return t


def all_gather_last_dim(t: torch.Tensor, group: Optional[dist.ProcessGroup] = None) -> torch.Tensor:
    """Concatenate every rank's [..., n] slice along the last dimension (rank order); identity without a process group."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return t
    parts = [torch.empty_like(t) for _ in range(dist.get_world_size(group))]
    dist.all_gather(parts, t.contiguous(), group=group)
    return torch.cat(parts, dim=-1)


class GatheredColumnParallelLinear(torch.nn.Module):
    """Tensor parallelism for an ACT-ORDER o_proj / down_proj, which `shard_rows` has to refuse (a row shard of an
    act-order layer no longer holds whole quantisation groups; the reference's engines replicate the scale tables and
    walk arbitrary g_idx instead, utils/marlin.py:296-305).  The layer is COLUMN-sharded (`shard_columns` keeps g_idx
    whole, so any act-order layer qualifies) and wrapped as

        x_shard [.., K/P] --all-gather--> x [.., K] --inner (N/P output features)--> y_shard --all-gather--> y [.., N]

    i.e. two all-gathers of activation-sized tensors instead of one all-reduce; every rank ends with the full output,
    exactly like RowParallelLinear, so the two are interchangeable inside a model."""

    def __init__(self, inner: torch.nn.Module, group: Optional[dist.ProcessGroup] = None, gather_input: bool = True):
        super().__init__()
        self.inner = inner
        self.group = group
        self.gather_input = gather_input

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.gather_input:
            x = all_gather_last_dim(x, self.group)
        return all_gather_last_dim(self.inner(x), self.group)


class FusedDecodeAllReduce:
    """Symmetric buffers for `b2q_decode_allreduce`: the row-parallel QuantLinear and its all-reduce in ONE kernel.

    One instance per TP group and device serves every row-parallel layer (calls are stream-ordered); layout per rank:
    f32 data[2][world][max_elems] | u32 flags (b2q_decode_allreduce_flag_bytes()), zero-initialised once.
    EXPERIMENTAL in round 1 (compiled, not yet validated on GPUs).
    """

    def __init__(self, device, max_elems: int = 8 * 8192, group: Optional[dist.ProcessGroup] = None):
        import ctypes

        import torch.distributed._symmetric_memory as symm_mem

        from ._lib import lib

        group = group if group is not None else dist.group.WORLD
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        if not 2 <= self.world <= 8:
            raise NotImplementedError("FusedDecodeAllReduce: 2..8 GPUs of one NVLink domain")
        self.max_elems = (max_elems + 31) // 32 * 32
        self.flag_offset = 2 * self.world * self.max_elems * 4
        nbytes = self.flag_offset + int(lib.b2q_decode_allreduce_flag_bytes())
        nbytes = (nbytes + 1023) // 1024 * 1024
        self.buf = symm_mem.empty(nbytes // 4, dtype=torch.int32, device=device)
        self.buf.zero_()
        self.hdl = symm_mem.rendezvous(self.buf, group.group_name)
        self._peers = (ctypes.c_void_p * self.world)(*[int(p) for p in self.hdl.buffer_ptrs])
        self.ctl = torch.zeros(4, dtype=torch.int32, device=device)  # {sequence, arrivals, status, -}
        torch.cuda.synchronize(device)
        dist.barrier(group)  # every rank's buffer is zeroed before anybody pushes into it

    def status(self) -> int:
        """0, or 1 + the rank of a peer whose flag never arrived within the kernel's 2 s bound (host sync; debugging)."""
        return int(self.ctl[2].item())


class RowParallelLinear(torch.nn.Module):
    """Wraps a row-sharded QuantLinear: forward(x_shard) -> all-reduced full output.

    reduce: None -> NCCL all-reduce; a `P2PAllReduce` -> our one-shot kernel after the matmul (decode-sized outputs);
    a `FusedDecodeAllReduce` -> matmul and all-reduce in one launch when the input has <= 8 tokens.
    """

    def __init__(self, inner: torch.nn.Module, group: Optional[dist.ProcessGroup] = None, reduce=None,
                 overlap_chunks: int = 1, overlap_min_tokens: int = 1024):
        super().__init__()
        self.inner = inner
        self.group = group
        self.reduce = reduce
        self.overlap_chunks = overlap_chunks
        self.overlap_min_tokens = overlap_min_tokens
        self._side = None

    def _forward_overlapped(self, x2: torch.Tensor) -> torch.Tensor:
        """Prefill-sized inputs: the token rows are cut into `overlap_chunks` blocks (multiples of the 256-row GEMM tile);
        the NCCL all-reduce of block c runs on a side stream while the shard's GEMM of block c + 1 runs on the caller's
        stream, so only the last block's collective is exposed.  Fork / join with events: CUDA-graph capturable.  OPT-IN
        (`overlap_chunks` > 1): the smaller GEMMs fill the SMs worse, NCCL competes for SMs with the GEMM it overlaps, and the
        blocks are concatenated afterwards, so it can be slower than one GEMM + one all-reduce."""
        M = x2.shape[0]
        cs = -(-M // self.overlap_chunks)
        cs = max(256, (cs + 255) // 256 * 256)
        cur = torch.cuda.current_stream(x2.device)
        if self._side is None:
            self._side = torch.cuda.Stream(device=x2.device)
        side = self._side
        parts = []
        for c0 in range(0, M, cs):
            yc = self.inner(x2[c0:c0 + cs])
            ev = torch.cuda.Event()
            ev.record(cur)
            side.wait_event(ev)
            with torch.cuda.stream(side):
                dist.all_reduce(yc, op=dist.ReduceOp.SUM, group=self.group)
            parts.append(yc)  # kept alive until the join below: no allocator reuse while the side stream still reads it
        cur.wait_stream(side)
        return torch.cat(parts, dim=0)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        tokens = x.numel() // x.shape[-1]
        if (self.overlap_chunks > 1 and tokens >= self.overlap_min_tokens and x.is_cuda and dist.is_available()
                and dist.is_initialized() and dist.get_world_size(self.group) > 1):
            y = self._forward_overlapped(x.reshape(-1, x.shape[-1]))
            return y.reshape(x.shape[:-1] + (y.shape[-1],))
        if isinstance(self.reduce, FusedDecodeAllReduce) and 1 <= tokens <= 8 and getattr(self.inner, "perm", 1) is None \
                and getattr(self.inner, "bits", 0) == 4 and not getattr(self.inner, "adapter", None):
            return self.inner.forward_allreduce(x, self.reduce)
        y = self.inner(x)
        if isinstance(self.reduce, P2PAllReduce) and y.numel() <= self.reduce.max_elems and y.numel() % 8 == 0:
            return self.reduce(y.contiguous())
        return all_reduce_sum_(y, self.group)
