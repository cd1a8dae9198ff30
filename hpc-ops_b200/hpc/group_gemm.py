"""Grouped FP8 GEMM operators (API of reference hpc/group_gemm.py) and the grouped bf16 GEMM of
fuse_moe_bf16 (no reference counterpart)."""
from typing import Optional as _Optional

import torch
from torch import Tensor

from . import _ops
from ._ffi import (check as _check_rc, lib as _lib, ptr as _ptr, require as _require,
                   stream_of as _stream_of)


def _scale_tile(avg: int) -> int:
    # The granule group_gemm_blockwise_fp8 reads the layout with (csrc/group_gemm_fp8.cu
    # scale_tile_from_avg). The reference's reformat entry (src/group_gemm/entry.cc:191-202) uses 64
    # for every avg > 48, which its GEMM does not for 65 <= avg <= 144.
    return int(_lib.hpc_scale_tile_from_avg(int(avg)))


def _check_common(x, weight, seqlens, cu_seqlens):
    _require(x.is_cuda and weight.is_cuda and seqlens.is_cuda and cu_seqlens.is_cuda,
             "x, weight, seqlens and cu_seqlens must be cuda tensors")
    _require(x.is_contiguous() and weight.is_contiguous(), "x and weight must be contiguous")
    _require(x.dtype == torch.float8_e4m3fn and weight.dtype == torch.float8_e4m3fn,
             "x and weight dtype must be fp8_e4m3")
    _require(seqlens.dtype == torch.int32 and cu_seqlens.dtype == torch.int32,
             "seqlens and cu_seqlens dtype must be int32")
    _require(seqlens.size(0) == weight.size(0), "seqlens and weight must share the same num_group")
    _require(x.size(1) == weight.size(2), "x and weight must share the same k")


def _group_gemm_fp8_impl(x, weight, seqlens, cu_seqlens, y_scale, num_seq_per_group_avg, output,
                         tma_desc, task_map_workspace):
    # reference src/group_gemm/entry.cc:14-105
    _check_common(x, weight, seqlens, cu_seqlens)
    _require(y_scale.is_cuda and y_scale.dtype == torch.float32, "y_scale must be a cuda float32 tensor")
    m, k = x.shape
    n = weight.size(1)
    y = output if output is not None else torch.empty((m, n), dtype=torch.bfloat16, device=x.device)
    _check_rc(_lib.hpc_group_gemm_fp8_async(
        _ptr(y), _ptr(x), _ptr(weight), _ptr(seqlens), _ptr(cu_seqlens), _ptr(y_scale), None, None,
        None, None, 0, weight.size(0), m, n, k, int(num_seq_per_group_avg), 1, 0, _stream_of(x)),
        "group_gemm_fp8")
    return y


def _cp_async_common(x, weight, y_scale, seqlens):
    # reference src/group_gemm/cp_async/entry.cc:46-52
    _require(x.is_cuda and weight.is_cuda, "inputs must be CUDA tensors")
    _require(x.is_contiguous() and weight.is_contiguous(), "inputs must be contiguous")
    _require(x.dtype == torch.float8_e4m3fn, "x must be float8_e4m3fn")
    _require(weight.dtype == torch.float8_e4m3fn, "weight must be float8_e4m3fn")
    _require(y_scale.dtype == torch.float32, "y_scale must be float32")
    _require(seqlens.size(0) <= 512, "num_group must be <= 512")
    _require(x.size(1) == weight.size(2), "x and weight must share the same k")


def _group_gemm_fp8_cp_async_impl(x, weight, y_scale, seqlens, cu_seqlens, tiles, cu_tiles,
                                  use_task_map=False):
    # reference src/group_gemm/cp_async/entry.cc:41-92; tiles / cu_tiles / use_task_map are the
    # reference's host-side schedule, not needed by the device-scheduled kernel
    _cp_async_common(x, weight, y_scale, seqlens)
    m, k = x.shape
    n = weight.size(1)
    g = seqlens.size(0)
    y = torch.empty((m, n), dtype=torch.bfloat16, device=x.device)
    _check_rc(_lib.hpc_group_gemm_fp8_multistage_async(
        _ptr(y), _ptr(x), _ptr(weight), _ptr(y_scale), _ptr(seqlens), _ptr(cu_seqlens), _ptr(tiles),
        _ptr(cu_tiles), None, 0, m, n, k, g, (m // g) if g else 0, 0, _stream_of(x)),
        "group_gemm_fp8_cp_async")
    return y


def _group_gemm_fp8_scatter_cp_async_impl(x, weight, y_scale, row_indices, seqlens, cu_seqlens,
                                          tiles, cu_tiles, use_task_map=False):
    # reference src/group_gemm/cp_async/entry.cc:94-142: x is a row pool, row i of the problem is
    # x[row_indices[i]]; output rows are in compact order
    _cp_async_common(x, weight, y_scale, seqlens)
    _require(row_indices.dtype == torch.int32, "row_indices must be int32")
    pool_rows, k = x.shape
    m = row_indices.numel()
    n = weight.size(1)
    g = seqlens.size(0)
    y = torch.empty((m, n), dtype=torch.bfloat16, device=x.device)
    scratch = torch.empty((m, k), dtype=torch.float8_e4m3fn, device=x.device)
    _check_rc(_lib.hpc_group_gemm_fp8_scatter_async(
        _ptr(y), _ptr(x), _ptr(weight), _ptr(y_scale), _ptr(row_indices), _ptr(seqlens),
        _ptr(cu_seqlens), _ptr(tiles), _ptr(cu_tiles), None, 0, m, n, k, g, (m // g) if g else 0, 0,
        _ptr(scratch), pool_rows, _stream_of(x)), "group_gemm_fp8_scatter_cp_async")
    return y


def _group_gemm_blockwise_fp8_impl(x, weight, seqlens, cu_seqlens, xscale, wscale,
                                   num_seq_per_group_avg, output, tma_desc, task_map_workspace):
    # reference src/group_gemm/entry.cc:107-178
    _check_common(x, weight, seqlens, cu_seqlens)
    _require(xscale.dtype == torch.float32 and wscale.dtype == torch.float32,
             "x_scale and w_scale dtype must be float32")
    _require(xscale.is_contiguous() and wscale.is_contiguous(), "scales must be contiguous")
    _require(wscale.size(2) % 4 == 0, "w_scale must be multiple of 4")
    m, k = x.shape
    n = weight.size(1)
    y = output if output is not None else torch.empty((m, n), dtype=torch.bfloat16, device=x.device)
    _check_rc(_lib.hpc_group_gemm_blockwise_fp8_async(
        _ptr(y), _ptr(x), _ptr(weight), _ptr(seqlens), _ptr(cu_seqlens), _ptr(xscale), _ptr(wscale),
        None, None, None, None, 0, weight.size(0), m, n, k, xscale.size(1), wscale.size(2),
        int(num_seq_per_group_avg), 1, 0, _stream_of(x)), "group_gemm_blockwise_fp8")
    return y


def _reformat_x_scale_impl(x_scale, seqlens, cu_seqlens, out_x_scale, num_seq_per_group_avg):
    # reference src/group_gemm/entry.cc:180-223
    _require(x_scale.is_cuda and seqlens.is_cuda and cu_seqlens.is_cuda, "tensors must be cuda")
    _require(x_scale.is_contiguous(), "x_scale tensor a must be contiguous")
    m, n = x_scale.shape
    tilem = _scale_tile(int(num_seq_per_group_avg))
    num_group = seqlens.size(0)
    _require((m // num_group) % tilem == 0,
             "The sparse pad length of x_scale for each group must be aligned to multiple of "
             "8/16/32/48/64 according to num_seq_per_group_avg")
    out = out_x_scale if out_x_scale is not None else torch.empty((n, m), dtype=x_scale.dtype,
                                                                  device=x_scale.device)
    _check_rc(_lib.hpc_reformat_x_scale_async(_ptr(out), _ptr(x_scale), _ptr(seqlens),
                                              _ptr(cu_seqlens), num_group, m, n, tilem,
                                              _stream_of(x_scale)), "reformat_x_scale")
    return out


_ops.define(
    "group_gemm_fp8(Tensor x, Tensor weight, Tensor seqlens, Tensor cu_seqlens, Tensor y_scale, "
    "int num_seq_per_group_avg, Tensor? output, Tensor? tma_desc, Tensor? task_map_workspace) -> "
    "(Tensor)")
_ops.impl("group_gemm_fp8", _group_gemm_fp8_impl, "CUDA")
_ops.define(
    "group_gemm_pertensor_fp8(Tensor x, Tensor weight, Tensor seqlens, Tensor cu_seqlens, Tensor "
    "y_scale, int num_seq_per_group_avg, Tensor? output, Tensor? tma_desc, Tensor? "
    "task_map_workspace) -> (Tensor)")
_ops.impl("group_gemm_pertensor_fp8", _group_gemm_fp8_impl, "CUDA")
_ops.define(
    "group_gemm_blockwise_fp8(Tensor x, Tensor weight, Tensor seqlens, Tensor cu_seqlens, Tensor "
    "xscale, Tensor wscale,"
    "int num_seq_per_group_avg, Tensor? output, Tensor? tma_desc, Tensor? task_map_workspace) -> "
    "(Tensor)")
_ops.impl("group_gemm_blockwise_fp8", _group_gemm_blockwise_fp8_impl, "CUDA")
_ops.define(
    "reformat_x_scale(Tensor x_scale, Tensor seqlens, Tensor cu_seqlens, "
    "Tensor? out_x_scale, int num_seq_per_group_avg) -> (Tensor)")
_ops.impl("reformat_x_scale", _reformat_x_scale_impl, "CUDA")


def reformat_x_scale(x_scale: Tensor, seqlens: Tensor, cu_seqlens: Tensor,
                     num_seq_per_group_avg: int, output: _Optional[Tensor] = None) -> Tensor:
    """Row-major DeepEP-style scales [total_seq_pad, k/128] -> the transposed, tile-compacted
    [k/128, total_seq_pad] layout `group_gemm_blockwise_fp8` reads (reference hpc/group_gemm.py:8-48)."""
    return torch.ops.hpc.reformat_x_scale(x_scale, seqlens, cu_seqlens, output, num_seq_per_group_avg)


def group_gemm_pertensor_fp8(x: Tensor, weight: Tensor, seqlens: Tensor, cu_seqlens: Tensor,
                             y_scale: Tensor, num_seq_per_group_avg: int = 32, output: Tensor = None,
                             tma_desc: Tensor = None, task_map_workspace: Tensor = None) -> Tensor:
    """Y[rows of g] = (X[rows of g] @ W[g]^T) * y_scale[g] -> bf16 (reference hpc/group_gemm.py:51-107)."""
    return torch.ops.hpc.group_gemm_pertensor_fp8(x, weight, seqlens, cu_seqlens, y_scale,
                                                  num_seq_per_group_avg, output, tma_desc,
                                                  task_map_workspace)


def group_gemm_fp8(x: Tensor, weight: Tensor, seqlens: Tensor, cu_seqlens: Tensor, y_scale: Tensor,
                   num_seq_per_group_avg: int = 32, output: Tensor = None, tma_desc: Tensor = None,
                   task_map_workspace: Tensor = None) -> Tensor:
    """Alias of group_gemm_pertensor_fp8 (reference hpc/group_gemm.py:110-131)."""
    return torch.ops.hpc.group_gemm_fp8(x, weight, seqlens, cu_seqlens, y_scale,
                                        num_seq_per_group_avg, output, tma_desc, task_map_workspace)


def group_gemm_blockwise_fp8(x: Tensor, weight: Tensor, seqlens: Tensor, cu_seqlens: Tensor,
                             x_scale: Tensor, w_scale: Tensor, num_seq_per_group_avg: int = 32,
                             output: Tensor = None, tma_desc: Tensor = None,
                             task_map_workspace: Tensor = None) -> Tensor:
    """128x128-blockwise-scaled grouped FP8 GEMM (reference hpc/group_gemm.py:134-197).
      x [total_seq, k] e4m3; weight [G, n, k] e4m3; x_scale f32 [k/128, total_seq_pad] (transposed,
      per-group columns padded to the tile of num_seq_per_group_avg); w_scale f32 [G, n/128, pad4(k/128)].
    Returns bf16 [total_seq, n]."""
    return torch.ops.hpc.group_gemm_blockwise_fp8(x, weight, seqlens, cu_seqlens, x_scale, w_scale,
                                                  num_seq_per_group_avg, output, tma_desc,
                                                  task_map_workspace)


@torch.library.register_fake("hpc::group_gemm_fp8")
def _group_gemm_fp8_fake(x, weight, seqlens, cu_seqlens, y_scale, num_seq_per_group_avg, output,
                         tma_desc, task_map_workspace):
    return torch.empty((x.shape[0], weight.shape[1]), dtype=torch.bfloat16, device=x.device)


@torch.library.register_fake("hpc::group_gemm_pertensor_fp8")
def _group_gemm_pertensor_fp8_fake(x, weight, seqlens, cu_seqlens, y_scale, num_seq_per_group_avg,
                                   output, tma_desc, task_map_workspace):
    return torch.empty((x.shape[0], weight.shape[1]), dtype=torch.bfloat16, device=x.device)


@torch.library.register_fake("hpc::group_gemm_blockwise_fp8")
def _group_gemm_blockwise_fp8_fake(x, weight, seqlens, cu_seqlens, xscale, wscale,
                                   num_seq_per_group_avg, output, tma_desc, task_map_workspace):
    return torch.empty((x.shape[0], weight.shape[1]), dtype=torch.bfloat16, device=x.device)

_ops.define(
    "group_gemm_fp8_cp_async(Tensor x, Tensor weight, Tensor y_scale, Tensor seqlens, Tensor "
    "cu_seqlens, Tensor tiles, Tensor cu_tiles, bool use_task_map=False) -> (Tensor)")
_ops.impl("group_gemm_fp8_cp_async", _group_gemm_fp8_cp_async_impl, "CUDA")
_ops.define(
    "group_gemm_fp8_scatter_cp_async(Tensor x, Tensor weight, Tensor y_scale, Tensor "
    "row_indices, Tensor seqlens, Tensor cu_seqlens, Tensor tiles, Tensor cu_tiles, "
    "bool use_task_map=False) -> (Tensor)")
_ops.impl("group_gemm_fp8_scatter_cp_async", _group_gemm_fp8_scatter_cp_async_impl, "CUDA")


@torch.library.register_fake("hpc::group_gemm_fp8_cp_async")
def _group_gemm_fp8_cp_async_fake(x, weight, y_scale, seqlens, cu_seqlens, tiles, cu_tiles,
                                  use_task_map=False):
    return torch.empty((x.shape[0], weight.shape[1]), dtype=torch.bfloat16, device=x.device)


@torch.library.register_fake("hpc::group_gemm_fp8_scatter_cp_async")
def _group_gemm_fp8_scatter_cp_async_fake(x, weight, y_scale, row_indices, seqlens, cu_seqlens,
                                          tiles, cu_tiles, use_task_map=False):
    return torch.empty((row_indices.shape[0], weight.shape[1]), dtype=torch.bfloat16,
                       device=x.device)


def _group_gemm_bf16_impl(x, weight, seqlens, cu_seqlens, output):
    for tt, name, dt in ((x, "x", torch.bfloat16), (weight, "weight", torch.bfloat16),
                         (seqlens, "seqlens", torch.int32), (cu_seqlens, "cu_seqlens", torch.int32)):
        _require(tt.dtype == dt, f"group_gemm_bf16: {name} must be {dt}, got {tt.dtype}")
        _require(tt.is_contiguous(), f"group_gemm_bf16: {name} must be contiguous")
    _require(x.dim() == 2 and weight.dim() == 3,
             "group_gemm_bf16: x must be [M, K] and weight [G, N, K]")
    m, k = x.shape
    g, n, k2 = weight.shape
    _require(k2 == k, f"group_gemm_bf16: weight K {k2} differs from x's {k}")
    _require(k % 128 == 0 and k > 0, f"group_gemm_bf16: K {k} must be a positive multiple of 128")
    _require(n % 128 == 0 and n > 0, f"group_gemm_bf16: N {n} must be a positive multiple of 128")
    _require(1 <= g <= 512, f"group_gemm_bf16: groups {g} not in [1, 512]")
    _require(tuple(seqlens.shape) == (g,) and tuple(cu_seqlens.shape) == (g + 1,),
             f"group_gemm_bf16: seqlens must be [{g}] and cu_seqlens [{g + 1}]")
    if output is not None:
        _require(output.dtype == torch.bfloat16 and tuple(output.shape) == (m, n)
                 and output.is_contiguous(),
                 f"group_gemm_bf16: output must be a contiguous bf16 tensor of shape [{m}, {n}]")
    for tt, name in ((x, "x"), (weight, "weight"), (seqlens, "seqlens"), (cu_seqlens, "cu_seqlens"),
                     (output, "output")):
        _require(tt is None or tt.is_cuda, f"group_gemm_bf16: {name} must be a CUDA tensor")
        _require(tt is None or tt.data_ptr() % 16 == 0,
                 f"group_gemm_bf16: {name} must be 16-byte aligned")
    y = output if output is not None else torch.empty((m, n), dtype=torch.bfloat16, device=x.device)
    if m == 0:
        return y
    _check_rc(_lib.hpc_group_gemm_bf16_async(_ptr(y), _ptr(x), _ptr(weight), _ptr(seqlens),
                                             _ptr(cu_seqlens), g, m, n, k, _stream_of(x)),
              "group_gemm_bf16")
    return y


_ops.define("group_gemm_bf16(Tensor x, Tensor weight, Tensor seqlens, Tensor cu_seqlens, Tensor? "
            "output) -> (Tensor)")
_ops.impl("group_gemm_bf16", _group_gemm_bf16_impl, "CUDA")


def group_gemm_bf16(x: Tensor, weight: Tensor, seqlens: Tensor, cu_seqlens: Tensor,
                    output: _Optional[Tensor] = None) -> Tensor:
    """Grouped bf16 GEMM: Y[rows of g] = X[rows of g] . weight[g]^T in one persistent sm_90a kernel.

    x [M, K] bf16 holds the rows of group g at cu_seqlens[g] .. cu_seqlens[g] + seqlens[g]
    (seqlens int32 [G], cu_seqlens int32 [G+1], as group_gemm_pertensor_fp8); weight [G, N, K]
    bf16. Y [M, N] bf16 = bf16_rn of the fp32-accumulated products; rows outside every group are
    not written. K and N multiples of 128, 1 <= G <= 512, contiguous 16-byte aligned tensors;
    otherwise RuntimeError before any launch. A caller-given output is written and returned. No
    allocation beyond the output and no host synchronisation: capturable in a CUDA graph."""
    return torch.ops.hpc.group_gemm_bf16(x, weight, seqlens, cu_seqlens, output)


@torch.library.register_fake("hpc::group_gemm_bf16")
def _group_gemm_bf16_fake(x, weight, seqlens, cu_seqlens, output):
    return output if output is not None else torch.empty((x.shape[0], weight.shape[1]),
                                                         dtype=torch.bfloat16, device=x.device)
