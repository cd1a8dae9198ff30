"""FusedMoE operators (API of reference hpc/fuse_moe.py).

Host prep mirrors the reference entries (src/fuse_moe/entry.cc:269-639): validation, tile table,
scratch allocation — except that the bf16 Gate-Up scratch is not allocated: this build fuses
SiLU*mul + FP8 re-quant into the Gate-Up GEMM epilogue.
"""
import torch
from torch import Tensor

from . import _ops
from ._ffi import check as _check_rc, lib as _lib, ptr as _ptr, stream_of as _stream_of


def _require(cond: bool, msg: str):
    if not cond:
        raise RuntimeError(msg)


def _aligned_size(avg: int) -> int:
    # reference src/fuse_moe/entry.cc:525-543
    for lim, val in ((8, 8), (16, 16), (32, 32), (48, 48), (64, 64), (96, 48), (128, 32), (144, 48)):
        if avg <= lim:
            return val
    return 64


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
