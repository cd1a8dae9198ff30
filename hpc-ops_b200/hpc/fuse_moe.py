"""FusedMoE operators (API of reference hpc/fuse_moe.py).

Host prep mirrors the reference entries (src/fuse_moe/entry.cc:269-639): validation, tile table,
scratch allocation — except that the bf16 Gate-Up scratch is not allocated: this build fuses
SiLU*mul + FP8 re-quant into the Gate-Up GEMM epilogue.

`moe_topk_gating` (no reference counterpart) turns the route GEMM's logits into the topk_ids /
topk_scale these operators consume, and `fuse_moe_bf16` (no reference counterpart either) runs the
expert layer of a bf16 model.
"""
from enum import IntEnum
from typing import Optional

import torch
from torch import Tensor

from . import _ops
from ._ffi import (check as _check_rc, lib as _lib, ptr as _ptr, require as _require,
                   stream_of as _stream_of)


def _aligned_size(avg: int) -> int:
    # reference src/fuse_moe/entry.cc:525-543; the rule the route kernel and the GEMMs use
    return int(_lib.hpc_scale_tile_from_avg(int(avg)))


def _check_moe_common(x, gate_up_weight, down_weight, topk_ids, topk_scale):
    _require(x.dtype == torch.float8_e4m3fn and gate_up_weight.dtype == torch.float8_e4m3fn
             and down_weight.dtype == torch.float8_e4m3fn,
             "x, gate_up_weight and down_weight dtype must be fp8_e4m3")
    _require(topk_ids.dtype == torch.int32, "topk_ids dtype must be int32")
    _require(topk_scale.dtype == torch.float32, "topk_scale dtype must be float32")
    for t, name in ((x, "x"), (gate_up_weight, "gate_up_weight"), (down_weight, "down_weight"),
                    (topk_ids, "topk_ids"), (topk_scale, "topk_scale")):
        _require(t.is_cuda, f"{name} tensor must be cuda")
        _require(t.is_contiguous(), f"{name} tensor must be contiguous")
    _require(x.size(0) == topk_ids.size(0), "x and topk_ids must share the same num_tokens")
    _require(topk_ids.shape == topk_scale.shape, "topk_ids and topk_scale must share the same shape")
    _require(x.size(1) == gate_up_weight.size(2), "x and weight must share the same k")
    _require(gate_up_weight.size(0) == down_weight.size(0),
             "gate_up_weight and down_weight must share the same num_expert")
    _require(topk_ids.size(1) <= 128, "num_topk must less than or equal to 128")


def _check_shared(shared_output, x):
    if shared_output is None:
        return
    _require(shared_output.is_cuda and shared_output.is_contiguous(),
             "shared_output tensor must be a contiguous cuda tensor")
    _require(shared_output.dtype == torch.bfloat16, "shared_output tensor dtype must be bfloat16")
    _require(tuple(shared_output.shape) == tuple(x.shape),
             "shared_output tensor shape must be same as x tensor")


def _out(output, num_tokens, hidden, device):
    if output is None:
        return torch.empty((num_tokens, hidden), dtype=torch.bfloat16, device=device)
    _require(output.size(0) == num_tokens and output.size(1) == hidden,
             "output shape must be [num_tokens, hidden_size]")
    _require(output.dtype == torch.bfloat16 and output.is_cuda, "output must be a cuda bf16 tensor")
    return output


def _fuse_moe_blockwise_impl(x, x_scale, gate_up_weight, gate_up_weight_scale, down_weight,
                             down_weight_scale, topk_ids, topk_scale, shared_output, rank_ep,
                             num_expert_total, output):
    _check_moe_common(x, gate_up_weight, down_weight, topk_ids, topk_scale)
    for t, name in ((x_scale, "x_scale"), (gate_up_weight_scale, "gate_up_weight_scale"),
                    (down_weight_scale, "down_weight_scale")):
        _require(t.is_cuda and t.is_contiguous() and t.dtype == torch.float32,
                 f"{name} must be a contiguous cuda float32 tensor")
    _require(x_scale.size(0) == x.size(0), "x_scale and x must share the same nun_tokens")
    _require(x_scale.size(1) == x.size(1) // 128, "x_scale must be per 128 blockwise quant")
    _require(gate_up_weight_scale.size(1) == gate_up_weight.size(1) // 128,
             "gate_up_weight must be per 128 blockwise quant")
    _require(gate_up_weight_scale.size(2) == (gate_up_weight.size(2) // 128 + 3) // 4 * 4,
             "gate_up_weight must be per 128 blockwise quant and must be aligned to 4")
    _require(down_weight_scale.size(1) == down_weight.size(1) // 128,
             "down_weight must be per 128 blockwise quant")
    _require(down_weight_scale.size(2) == (down_weight.size(2) // 128 + 3) // 4 * 4,
             "down_weight must be per 128 blockwise quant and must be aligned to 4")
    _check_shared(shared_output, x)
    y = _out(output, x.size(0), x.size(1), x.device)
    s = _blockwise_scratch(x, gate_up_weight, topk_ids, num_expert_total)
    _launch_blockwise(y, x, x_scale, gate_up_weight, gate_up_weight_scale, down_weight,
                      down_weight_scale, topk_ids, topk_scale, shared_output, rank_ep,
                      num_expert_total, s)
    return y


def _blockwise_scratch(x, gate_up_weight, topk_ids, num_expert_total):
    """Intermediate tensors of the blockwise pipeline, by stage:
      route    gate_up_input [rows, H] (gathered x rows, expert-major), gate_up_input_scale
               [H/128, num_padded] (transposed activation scales, each expert's columns padded to
               the scale granule), topk_pos, counts, cu_counts, tiles, cu_tiles;
      Gate-Up  down_input [rows, I] e4m3 and down_input_scale [I/128, num_padded] (same layout);
      Down     down_output [rows, H] bf16.
    Also returns num_padded (int)."""
    num_tokens, hidden = x.shape
    num_experts = gate_up_weight.size(0)
    inter = gate_up_weight.size(1) // 2
    num_topk = topk_ids.size(1)
    aligned = _aligned_size(num_tokens * num_topk // num_expert_total)
    rows = num_tokens * num_topk
    num_padded = (rows + num_expert_total * aligned + aligned - 1) // aligned * aligned
    dev = x.device
    i32 = dict(dtype=torch.int32, device=dev)
    return dict(
        gate_up_input=torch.empty((rows, hidden), dtype=torch.float8_e4m3fn, device=dev),
        gate_up_input_scale=torch.empty((hidden // 128, num_padded), dtype=torch.float32, device=dev),
        down_input=torch.empty((rows, inter), dtype=torch.float8_e4m3fn, device=dev),
        down_input_scale=torch.empty((inter // 128, num_padded), dtype=torch.float32, device=dev),
        down_output=torch.empty((rows, hidden), dtype=torch.bfloat16, device=dev),
        topk_pos=torch.empty((num_tokens, num_topk), **i32),
        counts=torch.empty((num_experts,), **i32),
        cu_counts=torch.empty((num_experts + 1,), **i32),
        tiles=torch.empty((num_experts,), **i32),
        cu_tiles=torch.empty((num_experts + 1,), **i32),
        num_padded=num_padded)


def _launch_blockwise(y, x, x_scale, gate_up_weight, gate_up_weight_scale, down_weight,
                      down_weight_scale, topk_ids, topk_scale, shared_output, rank_ep,
                      num_expert_total, s):
    """Enqueue the whole blockwise pipeline with the scratch `s` of _blockwise_scratch."""
    num_tokens, hidden = x.shape
    _check_rc(_lib.hpc_fuse_moe_blockwise_async(
        _ptr(y), _ptr(x), _ptr(x_scale), _ptr(s["gate_up_input"]), _ptr(s["gate_up_input_scale"]),
        None, _ptr(gate_up_weight), _ptr(gate_up_weight_scale), None, _ptr(s["down_input"]),
        _ptr(s["down_input_scale"]), _ptr(s["down_output"]), _ptr(down_weight),
        _ptr(down_weight_scale), None, _ptr(topk_ids), _ptr(topk_scale), _ptr(s["topk_pos"]),
        _ptr(s["counts"]), _ptr(s["cu_counts"]), _ptr(s["tiles"]), _ptr(s["cu_tiles"]),
        _ptr(shared_output), None, None, 0, 0, num_tokens, s["num_padded"], hidden,
        gate_up_weight.size(1), topk_ids.size(1), int(num_expert_total), gate_up_weight.size(0),
        gate_up_weight_scale.size(2), down_weight_scale.size(2), int(rank_ep), _stream_of(x)),
        "fuse_moe_blockwise")


def _fuse_moe_impl(x, gate_up_weight, down_weight, gate_up_scale, down_scale, act_and_mul_scale,
                   topk_ids, topk_scale, shared_output, rank_ep, num_expert_total, use_bf16_mul,
                   output):
    _check_moe_common(x, gate_up_weight, down_weight, topk_ids, topk_scale)
    for t, name in ((gate_up_scale, "gate_up_scale"), (down_scale, "down_scale"),
                    (act_and_mul_scale, "act_and_mul_scale")):
        _require(t.is_cuda and t.dtype == torch.float32, f"{name} must be a cuda float32 tensor")
    _check_shared(shared_output, x)
    num_tokens, hidden = x.shape
    num_experts = gate_up_weight.size(0)
    inter2 = gate_up_weight.size(1)
    num_topk = topk_ids.size(1)
    rows = num_tokens * num_topk
    dev = x.device
    y = _out(output, num_tokens, hidden, dev)
    i32 = dict(dtype=torch.int32, device=dev)
    gate_up_input = torch.empty((rows, hidden), dtype=torch.float8_e4m3fn, device=dev)
    down_input = torch.empty((rows, inter2 // 2), dtype=torch.float8_e4m3fn, device=dev)
    down_output = torch.empty((rows, hidden), dtype=torch.bfloat16, device=dev)
    topk_pos = torch.empty((num_tokens, num_topk), **i32)
    counts = torch.empty((num_experts,), **i32)
    cu_counts = torch.empty((num_experts + 1,), **i32)
    tiles = torch.empty((num_experts,), **i32)
    cu_tiles = torch.empty((num_experts + 1,), **i32)
    _check_rc(_lib.hpc_fuse_moe_async(
        _ptr(y), _ptr(x), _ptr(gate_up_input), None, _ptr(gate_up_weight), _ptr(gate_up_scale), None,
        _ptr(act_and_mul_scale), _ptr(down_input), _ptr(down_output), _ptr(down_weight),
        _ptr(down_scale), None, _ptr(topk_ids), _ptr(topk_scale), _ptr(topk_pos), _ptr(counts),
        _ptr(cu_counts), _ptr(tiles), _ptr(cu_tiles), _ptr(shared_output), None, None, 0, 0,
        num_tokens, hidden, inter2, num_topk, int(num_expert_total), num_experts, int(rank_ep),
        int(bool(use_bf16_mul)), _stream_of(x)), "fuse_moe")
    return y


def _count_and_gather_impl(x, topk_ids, num_expert, rank_ep, intermediate_size,
                           num_seq_per_group_avg):
    # reference src/fuse_moe/entry.cc:14-120 (returns the scratch tuple of the per-tensor pipeline)
    _require(x.is_cuda and topk_ids.is_cuda, "x and topk_ids must be cuda")
    _require(x.dtype == torch.float8_e4m3fn and topk_ids.dtype == torch.int32, "bad dtypes")
    num_seq, hidden = x.shape
    num_topk = topk_ids.size(1)
    rows = num_seq * num_topk
    dev = x.device
    i32 = dict(dtype=torch.int32, device=dev)
    gate_up_input = torch.empty((rows, hidden), dtype=torch.float8_e4m3fn, device=dev)
    gate_up_output = torch.empty((rows, intermediate_size), dtype=torch.bfloat16, device=dev)
    down_input = torch.empty((rows, intermediate_size // 2), dtype=torch.float8_e4m3fn, device=dev)
    down_output = torch.empty((rows, hidden), dtype=torch.bfloat16, device=dev)
    topk_pos = torch.empty((num_seq, num_topk), **i32)
    seqlens = torch.empty((num_expert,), **i32)
    cu_seqlens = torch.empty((num_expert + 1,), **i32)
    tiles = torch.empty((num_expert,), **i32)
    cu_tiles = torch.empty((num_expert + 1,), **i32)
    tmas = torch.empty((num_expert * 2 * 128,), dtype=torch.int8, device=dev)
    _check_rc(_lib.hpc_count_and_gather_async(
        _ptr(gate_up_input), None, None, None, _ptr(x), _ptr(topk_ids), _ptr(topk_pos),
        _ptr(seqlens), _ptr(cu_seqlens), None, None, _ptr(tiles), _ptr(cu_tiles), None, None,
        num_seq, hidden, int(intermediate_size), num_topk, int(num_expert), int(rank_ep),
        int(num_seq_per_group_avg), _stream_of(x)), "count_and_gather")
    return (gate_up_input, gate_up_output, down_input, down_output, topk_pos, seqlens, cu_seqlens,
            tiles, cu_tiles)


def _reduce_impl(x, topk_pos, topk_scale, shared_output):
    _require(x.is_cuda and x.dtype == torch.bfloat16 and x.is_contiguous(),
             "x must be a contiguous cuda bf16 tensor")
    _require(topk_pos.dtype == torch.int32 and topk_scale.dtype == torch.float32, "bad dtypes")
    num_seq, num_topk = topk_pos.shape
    y = torch.empty((num_seq, x.size(1)), dtype=torch.bfloat16, device=x.device)
    _check_rc(_lib.hpc_reduce_async(_ptr(y), _ptr(x), _ptr(topk_pos.contiguous()),
                                    _ptr(topk_scale.contiguous()), _ptr(shared_output), x.size(0),
                                    num_seq, x.size(1), num_topk, 0, _stream_of(x)), "reduce")
    return y


_ops.define(
    "count_and_gather(Tensor x, Tensor topk_ids, int num_expert, int rank_ep, int "
    "intermediate_size, int num_seq_per_group_avg"
    ") -> (Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor)")
_ops.impl("count_and_gather", _count_and_gather_impl, "CUDA")
_ops.define("reduce(Tensor x, Tensor topk_pos, Tensor topk_scale, Tensor ? shared_output) -> (Tensor)")
_ops.impl("reduce", _reduce_impl, "CUDA")
for _name in ("fuse_moe", "fuse_moe_pertensor_fp8"):
    _ops.define(
        _name + "(Tensor x, Tensor gate_up_weight, Tensor down_weight, Tensor gate_up_scale, "
        "Tensor down_scale, Tensor act_and_mul_scale, Tensor topk_ids, Tensor topk_scale, Tensor ? "
        "shared_output, int rank_ep, int num_expert_total, bool use_bf16_mul, Tensor ? output) -> "
        "(Tensor)")
    _ops.impl(_name, _fuse_moe_impl, "CUDA")
for _name in ("fuse_moe_blockwise", "fuse_moe_blockwise_fp8"):
    _ops.define(
        _name + "(Tensor x, Tensor x_scale, Tensor gate_up_weight, Tensor gate_up_weight_scale, "
        "Tensor down_weight, Tensor down_weight_scale, Tensor topk_ids, Tensor topk_scale, Tensor ? "
        "shared_output, int rank_ep, int num_expert_total, Tensor ? output) -> (Tensor)")
    _ops.impl(_name, _fuse_moe_blockwise_impl, "CUDA")


def count_and_gather(x: Tensor, topk_ids: Tensor, num_expert: int, rank_ep: int,
                     intermediate_size: int, num_seq_per_group_avg: int):
    """Route tokens to local experts and gather their rows (reference hpc/fuse_moe.py:8-85).
    Row order inside an expert is token order (deterministic)."""
    return torch.ops.hpc.count_and_gather(x, topk_ids, num_expert, rank_ep, intermediate_size,
                                          num_seq_per_group_avg)


def reduce(x: Tensor, topk_pos: Tensor, topk_scale: Tensor, shared_output: Tensor = None) -> Tensor:
    """y[t] = sum_k x[topk_pos[t,k]] * topk_scale[t,k] (+ shared_output[t]) (reference hpc/fuse_moe.py:88-133)."""
    return torch.ops.hpc.reduce(x, topk_pos, topk_scale, shared_output)


def fuse_moe(x: Tensor, gate_up_weight: Tensor, down_weight: Tensor, gate_up_scale: Tensor,
             down_scale: Tensor, act_and_mul_scale: Tensor, topk_ids: Tensor, topk_scale: Tensor,
             rank_ep: int, num_expert_total: int, use_bf16_mul: bool = True,
             shared_output: Tensor = None, output: Tensor = None) -> Tensor:
    """Run per-tensor FP8 FusedMoE (reference hpc/fuse_moe.py:136-166)."""
    return torch.ops.hpc.fuse_moe(x, gate_up_weight, down_weight, gate_up_scale, down_scale,
                                  act_and_mul_scale, topk_ids, topk_scale, shared_output, rank_ep,
                                  num_expert_total, use_bf16_mul, output)


def fuse_moe_pertensor_fp8(x: Tensor, gate_up_weight: Tensor, down_weight: Tensor,
                           gate_up_scale: Tensor, down_scale: Tensor, act_and_mul_scale: Tensor,
                           topk_ids: Tensor, topk_scale: Tensor, rank_ep: int, num_expert_total: int,
                           use_bf16_mul: bool = True, shared_output: Tensor = None) -> Tensor:
    """Run per-tensor FP8 FusedMoE (reference hpc/fuse_moe.py:169-199)."""
    return torch.ops.hpc.fuse_moe_pertensor_fp8(x, gate_up_weight, down_weight, gate_up_scale,
                                                down_scale, act_and_mul_scale, topk_ids, topk_scale,
                                                shared_output, rank_ep, num_expert_total,
                                                use_bf16_mul, None)


def fuse_moe_blockwise_fp8(x: Tensor, x_scale: Tensor, gate_up_weight: Tensor,
                           gate_up_weight_scale: Tensor, down_weight: Tensor,
                           down_weight_scale: Tensor, topk_ids: Tensor, topk_scale: Tensor,
                           rank_ep: int, num_expert_total: int, shared_output: Tensor = None) -> Tensor:
    """Run blockwise FP8 FusedMoE (reference hpc/fuse_moe.py:202-229)."""
    return torch.ops.hpc.fuse_moe_blockwise_fp8(x, x_scale, gate_up_weight, gate_up_weight_scale,
                                                down_weight, down_weight_scale, topk_ids, topk_scale,
                                                shared_output, rank_ep, num_expert_total, None)


def fuse_moe_blockwise(x: Tensor, x_scale: Tensor, gate_up_weight: Tensor,
                       gate_up_weight_scale: Tensor, down_weight: Tensor, down_weight_scale: Tensor,
                       topk_ids: Tensor, topk_scale: Tensor, rank_ep: int, num_expert_total: int,
                       shared_output: Tensor = None, output: Tensor = None) -> Tensor:
    """Run blockwise FP8 FusedMoE (reference hpc/fuse_moe.py:232-260)."""
    return torch.ops.hpc.fuse_moe_blockwise(x, x_scale, gate_up_weight, gate_up_weight_scale,
                                            down_weight, down_weight_scale, topk_ids, topk_scale,
                                            shared_output, rank_ep, num_expert_total, output)


def _moe_fake(x, output):
    return output if output is not None else torch.empty((x.shape[0], x.shape[1]),
                                                         dtype=torch.bfloat16, device=x.device)


@torch.library.register_fake("hpc::fuse_moe")
def _fuse_moe_fake(x, gate_up_weight, down_weight, gate_up_scale, down_scale, act_and_mul_scale,
                   topk_ids, topk_scale, shared_output, rank_ep, num_expert_total, use_bf16_mul,
                   output):
    return _moe_fake(x, output)


@torch.library.register_fake("hpc::fuse_moe_pertensor_fp8")
def _fuse_moe_pertensor_fp8_fake(x, gate_up_weight, down_weight, gate_up_scale, down_scale,
                                 act_and_mul_scale, topk_ids, topk_scale, shared_output, rank_ep,
                                 num_expert_total, use_bf16_mul, output):
    return _moe_fake(x, output)


@torch.library.register_fake("hpc::fuse_moe_blockwise")
def _fuse_moe_blockwise_fake(x, x_scale, gate_up_weight, gate_up_weight_scale, down_weight,
                             down_weight_scale, topk_ids, topk_scale, shared_output, rank_ep,
                             num_expert_total, output):
    return _moe_fake(x, output)


@torch.library.register_fake("hpc::fuse_moe_blockwise_fp8")
def _fuse_moe_blockwise_fp8_fake(x, x_scale, gate_up_weight, gate_up_weight_scale, down_weight,
                                 down_weight_scale, topk_ids, topk_scale, shared_output, rank_ep,
                                 num_expert_total, output):
    return _moe_fake(x, output)


@torch.library.register_fake("hpc::reduce")
def _reduce_fake(x, topk_pos, topk_scale, shared_output):
    return torch.empty((topk_pos.shape[0], x.shape[1]), dtype=torch.bfloat16, device=x.device)


MAX_MOE_EXPERTS = 512
MAX_MOE_TOPK = 128


def _check_bf16(x, gate_up_weight, down_weight, topk_ids, topk_scale, num_expert_total,
                shared_output, output):
    """fuse_moe_bf16's limits, checked before any device work; returns (T, H, I, E_local, k)."""
    for t, name, dt in ((x, "x", torch.bfloat16), (gate_up_weight, "gate_up_weight", torch.bfloat16),
                        (down_weight, "down_weight", torch.bfloat16),
                        (topk_ids, "topk_ids", torch.int32), (topk_scale, "topk_scale", torch.float32)):
        _require(t.dtype == dt, f"fuse_moe_bf16: {name} must be {dt}, got {t.dtype}")
        _require(t.is_contiguous(), f"fuse_moe_bf16: {name} must be contiguous")
    _require(x.dim() == 2 and gate_up_weight.dim() == 3 and down_weight.dim() == 3
             and topk_ids.dim() == 2,
             "fuse_moe_bf16: x [T, H], gate_up_weight [E, 2I, H], down_weight [E, H, I] and "
             "topk_ids [T, k] have the wrong number of dimensions")
    T, H = x.shape
    E, I2, H2 = gate_up_weight.shape
    I = I2 // 2
    _require(H % 128 == 0 and H > 0, f"fuse_moe_bf16: hidden {H} must be a positive multiple of 128")
    _require(H2 == H, f"fuse_moe_bf16: gate_up_weight hidden {H2} differs from x's {H}")
    _require(I2 % 256 == 0 and I2 > 0,
             f"fuse_moe_bf16: gate_up_weight rows {I2} must be 2 * I with I a positive multiple of 128")
    _require(tuple(down_weight.shape) == (E, H, I),
             f"fuse_moe_bf16: down_weight must be [{E}, {H}, {I}], got {tuple(down_weight.shape)}")
    _require(1 <= E <= MAX_MOE_EXPERTS,
             f"fuse_moe_bf16: local experts {E} not in [1, {MAX_MOE_EXPERTS}]")
    _require(num_expert_total >= E,
             f"fuse_moe_bf16: num_expert_total {num_expert_total} below the {E} local experts")
    _require(topk_ids.size(0) == T and tuple(topk_scale.shape) == tuple(topk_ids.shape),
             f"fuse_moe_bf16: topk_ids and topk_scale must be [{T}, k]")
    k = topk_ids.size(1)
    _require(1 <= k <= MAX_MOE_TOPK, f"fuse_moe_bf16: num_topk {k} not in [1, {MAX_MOE_TOPK}]")
    for t, name in ((shared_output, "shared_output"), (output, "output")):
        if t is not None:
            _require(t.dtype == torch.bfloat16 and tuple(t.shape) == (T, H) and t.is_contiguous(),
                     f"fuse_moe_bf16: {name} must be a contiguous bf16 tensor of shape [{T}, {H}]")
    for t, name in ((x, "x"), (gate_up_weight, "gate_up_weight"), (down_weight, "down_weight"),
                    (topk_ids, "topk_ids"), (topk_scale, "topk_scale"),
                    (shared_output, "shared_output"), (output, "output")):
        _require(t is None or t.is_cuda, f"fuse_moe_bf16: {name} must be a CUDA tensor")
        _require(t is None or t.device == x.device, f"fuse_moe_bf16: {name} must be on x's device")
        _require(t is None or t.data_ptr() % 16 == 0, f"fuse_moe_bf16: {name} must be 16-byte aligned")
    return T, H, I, E, k


def _bf16_scratch(x, gate_up_weight, topk_ids):
    """Intermediate tensors of the bf16 pipeline, by stage:
      route    gate_up_input [rows, H] (gathered x rows, expert-major, token order inside an
               expert), topk_pos [T, k], counts [E], cu_counts [E+1], tiles [E] (128-row m-tiles
               per expert), cu_tiles [E+1];
      Gate-Up  down_input [rows, I] bf16 (silu(g) * u);
      Down     down_output [rows, H] bf16.
    rows = T * k (an upper bound: ids of other ranks take no row)."""
    num_tokens, hidden = x.shape
    num_experts = gate_up_weight.size(0)
    inter = gate_up_weight.size(1) // 2
    num_topk = topk_ids.size(1)
    rows = num_tokens * num_topk
    dev = x.device
    i32 = dict(dtype=torch.int32, device=dev)
    return dict(
        gate_up_input=torch.empty((rows, hidden), dtype=torch.bfloat16, device=dev),
        down_input=torch.empty((rows, inter), dtype=torch.bfloat16, device=dev),
        down_output=torch.empty((rows, hidden), dtype=torch.bfloat16, device=dev),
        topk_pos=torch.empty((num_tokens, num_topk), **i32),
        counts=torch.empty((num_experts,), **i32),
        cu_counts=torch.empty((num_experts + 1,), **i32),
        tiles=torch.empty((num_experts,), **i32),
        cu_tiles=torch.empty((num_experts + 1,), **i32))


def _launch_bf16(y, x, gate_up_weight, down_weight, topk_ids, topk_scale, shared_output, rank_ep,
                 num_expert_total, s):
    """Enqueue the whole bf16 pipeline with the scratch `s` of _bf16_scratch."""
    num_tokens, hidden = x.shape
    _check_rc(_lib.hpc_fuse_moe_bf16_async(
        _ptr(y), _ptr(x), _ptr(s["gate_up_input"]), _ptr(gate_up_weight), _ptr(s["down_input"]),
        _ptr(s["down_output"]), _ptr(down_weight), _ptr(topk_ids), _ptr(topk_scale),
        _ptr(s["topk_pos"]), _ptr(s["counts"]), _ptr(s["cu_counts"]), _ptr(s["tiles"]),
        _ptr(s["cu_tiles"]), _ptr(shared_output), num_tokens, hidden, gate_up_weight.size(1) // 2,
        topk_ids.size(1), int(num_expert_total), gate_up_weight.size(0), int(rank_ep),
        _stream_of(x)), "fuse_moe_bf16")


def _fuse_moe_bf16_impl(x, gate_up_weight, down_weight, topk_ids, topk_scale, rank_ep,
                        num_expert_total, shared_output, output):
    T, H, _, _, _ = _check_bf16(x, gate_up_weight, down_weight, topk_ids, topk_scale,
                                num_expert_total, shared_output, output)
    y = output if output is not None else torch.empty((T, H), dtype=torch.bfloat16, device=x.device)
    if T == 0:
        return y
    s = _bf16_scratch(x, gate_up_weight, topk_ids)
    _launch_bf16(y, x, gate_up_weight, down_weight, topk_ids, topk_scale, shared_output, rank_ep,
                 num_expert_total, s)
    return y


_ops.define(
    "fuse_moe_bf16(Tensor x, Tensor gate_up_weight, Tensor down_weight, Tensor topk_ids, Tensor "
    "topk_scale, int rank_ep, int num_expert_total, Tensor? shared_output, Tensor? output) -> "
    "(Tensor)")
_ops.impl("fuse_moe_bf16", _fuse_moe_bf16_impl, "CUDA")


def fuse_moe_bf16(x: Tensor, gate_up_weight: Tensor, down_weight: Tensor, topk_ids: Tensor,
                  topk_scale: Tensor, rank_ep: int, num_expert_total: int,
                  shared_output: Optional[Tensor] = None, output: Optional[Tensor] = None) -> Tensor:
    """bf16 FusedMoE: the expert layer of a bf16 MoE model in four sm_90a kernels (route, fused
    Gate-Up GEMM + SiLU*mul, Down GEMM, top-k reduce) on the current stream.

    x [T, H] bf16; gate_up_weight [E_local, 2I, H] bf16 (gate rows, then up rows, as fuse_moe* and
    vLLM's w13); down_weight [E_local, H, I] bf16; topk_ids int32 / topk_scale float32 [T, k] as
    moe_topk_gating returns them. This rank owns experts [rank_ep E_local, (rank_ep+1) E_local) of
    num_expert_total; other ids contribute nothing. Per routed row r of local expert e, with fp32
    accumulation:
      1. g_j = bf16(sum_h x[h] W13[e, j, h]), u_j = bf16(sum_h x[h] W13[e, I+j, h]);
      2. a_j = bf16(silu(g_j) * u_j), the product in fp32 (silu x / (1 + exp(-x)) with fast
         exp and division, as the FP8 epilogue);
      3. d = bf16(sum_j a_j W2[e, :, j]);
      4. y[t] = bf16(sum_k topk_scale[t, k] d[pos[t, k]] (+ shared_output[t])), fp32 sums in k order.
    Rows inside an expert are in token order, so two calls give the same bits.

    Limits: H and I multiples of 128, 1 <= E_local <= 512, 1 <= k <= 128, contiguous 16-byte
    aligned tensors on one device; otherwise RuntimeError before any launch. T = 0 returns without a
    launch. shared_output [T, H] bf16 is added in the reduce; a caller-given output [T, H] bf16 is
    written and returned. Scratch is allocated by torch's caching allocator, the launcher neither
    allocates nor synchronises with the host: the call can be captured in a CUDA graph."""
    return torch.ops.hpc.fuse_moe_bf16(x, gate_up_weight, down_weight, topk_ids, topk_scale,
                                       int(rank_ep), int(num_expert_total), shared_output, output)


@torch.library.register_fake("hpc::fuse_moe_bf16")
def _fuse_moe_bf16_fake(x, gate_up_weight, down_weight, topk_ids, topk_scale, rank_ep,
                        num_expert_total, shared_output, output):
    return _moe_fake(x, output)


class GatingScore(IntEnum):
    """How moe_topk_gating turns a router logit into an expert score."""
    SOFTMAX = 0
    SIGMOID = 1


MAX_GATING_EXPERTS = 512
MAX_GATING_TOPK = 16


def _check_gating(router_logits, topk, scoring, correction_bias, num_expert_group, topk_group,
                  topk_ids, topk_weights):
    """The launcher's limits, checked before any device work; returns (num_tokens, num_experts)."""
    x = router_logits
    _require(x.dim() == 2, f"moe_topk_gating: router_logits must be 2-D [T, E], got {tuple(x.shape)}")
    _require(x.dtype in (torch.float32, torch.bfloat16),
             f"moe_topk_gating: router_logits must be float32 or bfloat16, got {x.dtype}")
    T, E = x.shape
    _require(x.stride(1) == 1 or E == 1, "moe_topk_gating: router_logits rows must be contiguous")
    _require(1 <= E <= MAX_GATING_EXPERTS,
             f"moe_topk_gating: number of experts {E} outside [1, {MAX_GATING_EXPERTS}]")
    _require(1 <= topk <= min(MAX_GATING_TOPK, E),
             f"moe_topk_gating: topk {topk} outside [1, min({MAX_GATING_TOPK}, {E})]")
    _require(int(scoring) in (0, 1), f"moe_topk_gating: unknown scoring {scoring}")
    G = num_expert_group
    _require(G >= 1 and E % G == 0,
             f"moe_topk_gating: num_expert_group {G} must be positive and divide the {E} experts")
    _require(1 <= topk_group <= G,
             f"moe_topk_gating: topk_group {topk_group} outside [1, num_expert_group {G}]")
    _require(topk <= topk_group * (E // G),
             f"moe_topk_gating: topk {topk} exceeds the {topk_group * (E // G)} experts of "
             f"topk_group {topk_group} groups")
    esize = x.element_size()
    if T > 1:
        _require(x.stride(0) >= E and x.stride(0) * esize % 16 == 0,
                 f"moe_topk_gating: row stride {x.stride(0)} elements must be at least the {E} "
                 "experts and a multiple of 16 bytes")
    if correction_bias is not None:
        _require(correction_bias.dtype == torch.float32 and correction_bias.dim() == 1
                 and correction_bias.numel() == E and correction_bias.is_contiguous(),
                 f"moe_topk_gating: correction_bias must be a contiguous float32 tensor of {E} "
                 "values")
        _require(G == 1 or E // G >= 2,
                 "moe_topk_gating: a correction bias with groups needs at least 2 experts per "
                 "group (the group score is the sum of its top-2 keys)")
    for t, name, dt in ((topk_ids, "topk_ids", torch.int32), (topk_weights, "topk_weights", torch.float32)):
        if t is not None:
            _require(t.dtype == dt and tuple(t.shape) == (T, topk) and t.is_contiguous(),
                     f"moe_topk_gating: {name} must be a contiguous {dt} tensor of shape "
                     f"[{T}, {topk}]")
    _require(x.is_cuda, "moe_topk_gating: router_logits must be a CUDA tensor")
    for t, name in ((correction_bias, "correction_bias"), (topk_ids, "topk_ids"),
                    (topk_weights, "topk_weights")):
        _require(t is None or t.device == x.device,
                 f"moe_topk_gating: {name} must be on the device of router_logits")
    _require(x.data_ptr() % 16 == 0, "moe_topk_gating: router_logits must be 16-byte aligned")
    return T, E


def _moe_topk_gating_impl(router_logits, topk, scoring, renormalize, correction_bias,
                          num_expert_group, topk_group, routed_scaling_factor, topk_ids,
                          topk_weights):
    T, E = _check_gating(router_logits, topk, scoring, correction_bias, num_expert_group,
                         topk_group, topk_ids, topk_weights)
    dev = router_logits.device
    if topk_ids is None:
        topk_ids = torch.empty((T, topk), dtype=torch.int32, device=dev)
    if topk_weights is None:
        topk_weights = torch.empty((T, topk), dtype=torch.float32, device=dev)
    if T == 0:
        return topk_ids, topk_weights
    _check_rc(_lib.hpc_moe_topk_gating_async(
        _ptr(router_logits), _ptr(correction_bias), _ptr(topk_ids), _ptr(topk_weights), T, E,
        0 if router_logits.dtype == torch.float32 else 1, int(topk), int(scoring),
        int(bool(renormalize)), int(num_expert_group), int(topk_group), router_logits.stride(0),
        float(routed_scaling_factor), _stream_of(router_logits)), "moe_topk_gating")
    return topk_ids, topk_weights


_ops.define(
    "moe_topk_gating(Tensor router_logits, int topk, int scoring, bool renormalize, Tensor? "
    "correction_bias, int num_expert_group, int topk_group, float routed_scaling_factor, Tensor? "
    "topk_ids, Tensor? topk_weights) -> (Tensor, Tensor)")
_ops.impl("moe_topk_gating", _moe_topk_gating_impl, "CUDA")


def moe_topk_gating(router_logits: Tensor, topk: int, scoring: GatingScore = GatingScore.SOFTMAX,
                    renormalize: bool = True, correction_bias: Optional[Tensor] = None,
                    num_expert_group: int = 1, topk_group: int = 1,
                    routed_scaling_factor: float = 1.0, topk_ids: Optional[Tensor] = None,
                    topk_weights: Optional[Tensor] = None) -> tuple:
    """Router logits -> (topk_ids int32 [T, topk], topk_weights float32 [T, topk]), the
    topk_ids / topk_scale of fuse_moe*, in one sm_90a kernel.

    router_logits [T, E] float32 or bfloat16 with contiguous rows and any 16-byte row stride, so
    a column slice `logits[:, :E]` of a wider (padded) route-GEMM output is read in place.
    Per token row, in fp32 (x_e = float(logits[t, e])):

    1. Score s_e: SOFTMAX exp(x_e - max x) / sum_j exp(x_j - max x) over all E; SIGMOID
       1 / (1 + exp(-x_e)).
    2. Selection key c_e: x_e for SOFTMAX without a bias (the order of s_e, exactly: logits that
       round to one fp32 score do not tie); otherwise s_e + correction_bias[e].
    3. num_expert_group G > 1 (E % G == 0): group g is experts [g E/G, (g+1) E/G). Its score is
       the sum of its top-2 keys with a bias, its max key without (vLLM's grouped_topk rule); the
       topk_group best groups, by (score desc, group id asc), stay eligible.
    4. The topk eligible experts in the order (key desc, id asc), NaN below -inf: every row's ids
       are distinct and in [0, E) for any input (its weights are unspecified when it holds NaN),
       and a -inf key is never chosen while a finite one is available.
    5. Weights w_i = s_{id_i} (the unbiased score); with renormalize, w_i /= sum_i w_i summed in
       rank order; then w_i *= routed_scaling_factor.
    6. Outputs in rank order. Caller-given topk_ids / topk_weights (contiguous, [T, topk]) are
       written in place and returned.

    Limits: 1 <= E <= 512, 1 <= topk <= min(16, E), topk_group <= G, topk <= topk_group E / G,
    groups of at least 2 experts with a bias, 16-byte aligned logits. T = 0 returns empty tensors
    without a launch. No allocation beyond the outputs and no host synchronisation: the call can
    be captured in a CUDA graph, and it chains to the following fuse_moe* launch by programmatic
    dependent launch."""
    return torch.ops.hpc.moe_topk_gating(router_logits, int(topk), int(scoring), bool(renormalize),
                                         correction_bias, int(num_expert_group), int(topk_group),
                                         float(routed_scaling_factor), topk_ids, topk_weights)


@torch.library.register_fake("hpc::moe_topk_gating")
def _moe_topk_gating_fake(router_logits, topk, scoring, renormalize, correction_bias,
                          num_expert_group, topk_group, routed_scaling_factor, topk_ids,
                          topk_weights):
    T = router_logits.shape[0]
    dev = router_logits.device
    ids = topk_ids if topk_ids is not None else torch.empty((T, topk), dtype=torch.int32, device=dev)
    w = (topk_weights if topk_weights is not None
         else torch.empty((T, topk), dtype=torch.float32, device=dev))
    return ids, w
