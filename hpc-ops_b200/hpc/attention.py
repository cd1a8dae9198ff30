"""Attention operators of the hot path (API of reference hpc/attention.py).

Implemented in this build (sm_90a):
  * attention_decode_fp8            — quant_type QPERTOKEN_PERHEAD_KPERTENSOR_VPERTENSOR and
                                      QPERTOKEN_PERHEAD_KPERTOKEN_PERHEAD_VPERHEAD (in-cache k scales)
  * attention_decode_bf16           — pages of 16 / 32 / 64 tokens, mtp 0..4
  * attention_decode_mla_bf16       — absorbed MLA (576 / 512 latent head) over a paged bf16 cache
  * attention_with_kvcache_blocksparse_prefill_fp8 / attention_with_kvcache_prefill_fp8 (dense)
  * attention_prefill_bf16 (varlen causal self-attention on contiguous q/k/v) and
    attention_with_kvcache_prefill_bf16 (causal, chunked, prefill over the paged bf16 cache,
    pages of 16 / 32 / 64 tokens)
  * attention_prefill_mla_bf16      — un-absorbed MLA prefill (192-wide q / k with a head-shared
                                      k_pe, 128-wide v), varlen, bottom-right causal
  * get_attention_decode_task_workspace / assign_attention_decode_task (CPU and CUDA)
  * print_attention_decode_task
The host side does what the reference's torch entry does (validation, scratch allocation, stride
extraction: reference src/attention/entry.cc:569-817) and then calls the C-ABI launcher.
"""
from enum import Enum as _Enum
from typing import Optional as _Optional

import torch
from torch import Tensor

from . import _ffi, _ops
from ._ffi import (check as _check_rc, lib as _lib, ptr as _ptr, require as _require,
                   stream_of as _stream_of)


class QuantType(_Enum):
    QPERTOKEN_PERHEAD_KPERTOKEN_PERHEAD_VPERHEAD = 0
    QPERTOKEN_PERHEAD_KPERTENSOR_VPERTENSOR = 1
    QPERTENSOR_KPERTENSOR_VPERTENSOR = 2
    QPERTOKEN_PERHEAD_KPERTOKEN_PERHEAD_VPERHEAD_QKHADAMARD = 3


# Scheduler constants of the decode kernels: 128-key tiles (two m64 wgmma halves), one persistent
# CTA per SM for every num_seq_q. Same values the reference reserves for major 10
# (reference src/attention/decode/sched_task_info.h:35-36, src/attention/entry.cc:736-742).
_TILE_N = 128
_CTA_PER_SM = 1
_TASK_BYTES = 48
_TASK_INTS = 12


_WORKSPACE_TEMPLATES = {}  # (device, geometry) -> zeroed task-map workspace with its header written


def _num_total_ctas(device=None) -> int:
    return _ffi.sm_count(device) * _CTA_PER_SM


# --------------------------------------------------------------------------------------------
# torch.ops.hpc.* implementations
# --------------------------------------------------------------------------------------------
def _attention_decode_fp8_impl(
    q, kcache, vcache, block_ids, num_seq_kvcache, qscale, kscale, vscale, mtp, new_kv_included,
    quant_type, use_splitk, task_map, split_flag, output,
):
    y, args, _keep = _decode_fp8_prepare(
        q, kcache, vcache, block_ids, num_seq_kvcache, qscale, kscale, vscale, mtp,
        new_kv_included, quant_type, use_splitk, task_map, split_flag, output)
    _check_rc(_lib.hpc_attention_decode_fp8_async(*args), "attention_decode_fp8")
    return y


def _decode_output(output, q, rows, num_head_q):
    """The decode output: a new [rows, num_head_q, 128] bf16 tensor, or the caller's `output`
    once checked. The split-k combine stores 8 bytes per lane (the attention kernel's direct write
    of an unsplit pair: 2) at y + row * y.stride(0) + head * 128, so rows may be strided (a view
    into a wider buffer, e.g. a fused output) but must hold [num_head_q, 128] contiguously, and
    the base and the row stride are kept 16-byte aligned."""
    if output is None:
        return torch.empty((rows, num_head_q, 128), dtype=torch.bfloat16, device=q.device)
    _require(output.is_cuda and output.device == q.device, "output tensor must be cuda, on q's device")
    _require(output.dtype == torch.bfloat16, "output dtype must be bfloat16")
    _require(tuple(output.shape) == (rows, num_head_q, 128),
             "output must have shape [num_batch * num_seq_q, num_head_q, 128]")
    _require(output.stride(2) == 1 and output.stride(1) == 128
             and (rows == 1 or output.stride(0) >= num_head_q * 128),
             "output rows must be [num_head_q, 128] contiguous and must not overlap")
    _require(output.data_ptr() % 16 == 0 and (rows == 1 or output.stride(0) % 8 == 0),
             "output and its row stride must be 16-byte aligned")
    return output


def _decode_fp8_prepare(
    q, kcache, vcache, block_ids, num_seq_kvcache, qscale, kscale, vscale, mtp, new_kv_included,
    quant_type, use_splitk, task_map, split_flag, output,
):
    """Validate, allocate scratch and marshal the C-ABI argument tuple.
    Returns (y, args, keepalive)."""
    # validation mirrors reference src/attention/entry.cc:580-616
    _require(q.is_cuda, "q tensor must be cuda")
    _require(kcache.is_cuda and vcache.is_cuda, "kv cache tensors must be cuda")
    _require(block_ids.is_cuda, "block_ids tensor must be cuda")
    _require(block_ids.is_contiguous(), "block_ids tensor must be contiguous")
    _require(num_seq_kvcache.is_contiguous(), "num_seq_kvcache tensor must be contiguous")
    _require(q.dtype == torch.float8_e4m3fn, "q dtype must be fp8_e4m3fn")
    _require(kcache.element_size() == 1, "kcache tensor element type size must be fp8_e4m3")
    _require(vcache.element_size() == 1, "vcache tensor element type size must be fp8_e4m3")
    _require(block_ids.dtype == torch.int32, "block_ids dtype must be int32")
    _require(num_seq_kvcache.dtype == torch.int32, "num_seq_kvcache dtype must be int32")
    _require(mtp in (0, 1, 2, 3), "we only support mtp 0, 1, 2, 3.")

    num_batch = num_seq_kvcache.size(0)
    num_seq_q = q.size(0) // num_batch
    _require(num_seq_q == mtp + 1, "every request num_seq_q must be mtp + 1")
    num_head_q = q.size(1)
    num_dim_qk = q.size(2)
    _require(num_dim_qk == 128, "we only support head dim 128.")
    num_kvcache_blocks = kcache.size(0)
    block_size = kcache.size(1)
    _require(block_size == 64, "kvcache paged blocksize must be 64.")
    num_head_k = kcache.size(2)
    num_head_v = vcache.size(2)
    num_dim_v = vcache.size(3)
    num_seq_max_blocks = block_ids.size(1)
    heads_per_group = num_head_q // num_head_k
    _require(heads_per_group in (4, 8), "we only support num_head_q / num_head_k == 4 or 8.")
    _require(q.stride(2) == 1 and q.stride(1) == num_dim_qk, "q must be contiguous in (head, dim)")
    _require(kcache.stride(3) == 1 and vcache.stride(3) == 1, "kv cache innermost dim must be contiguous")
    _require(qscale.dtype == torch.float32 and vscale.dtype == torch.float32, "scales must be float32")
    _require(int(quant_type) in (0, 1), "attention_decode_fp8 supports quant_type 0 and 1")
    if int(quant_type) == 0:
        # per-token k scales: fp32 words in the cache allocation's extra rows, logical shape
        # [blocks, bs/32, Hkv, D/4] f32, passed as an fp8 view or as f32; they share the cache's
        # strides (reference src/attention/entry.cc:245-253, tests/..qkpertoken..fp8.py:340-385)
        ks_unit = 4 // kscale.element_size()  # strides in elements -> floats
        _require(kscale.element_size() in (1, 4) and kscale.dim() == 4, "kscale must be [blocks, bs/32, Hkv, D/4] f32 (or its fp8 view)")
        for i in range(3):
            _require(kscale.stride(i) * kscale.element_size() == kcache.stride(i),
                     "k scale rows must be the extra rows of the kcache allocation (same strides)")
        _require(kscale.stride(3) == 1 and kscale.data_ptr() % 4 == 0 and ks_unit >= 1, "bad kscale layout")
        _require(vscale.numel() == num_head_k, "vscale must hold one scale per kv head")

    y = _decode_output(output, q, num_batch * num_seq_q, num_head_q)

    num_total_ctas = _num_total_ctas(q.device)
    if task_map is None:
        # The decode kernels are task-map driven. Without a caller-provided map we schedule on
        # the device right here (this build has no counterpart of the reference's static split-k
        # path, reference src/attention/entry.cc:649-652).
        task_map = get_attention_decode_task_workspace(
            num_batch, int(num_seq_max_blocks) * block_size + num_seq_q, num_head_k,
            min_process_len=512, device=q.device)
        _assign_task_cuda(num_seq_kvcache, num_head_k, num_seq_q, new_kv_included, 512, task_map)

    splitk = num_total_ctas
    pad_heads_per_group = (heads_per_group + 7) // 8 * 8
    lse = torch.empty((num_batch, splitk, num_head_k, num_seq_q, pad_heads_per_group),
                      dtype=torch.float32, device=q.device)
    split_out = torch.empty((num_batch, splitk, num_seq_q, num_head_q, num_dim_v),
                            dtype=torch.float32, device=q.device)

    args = (
        _ptr(y), _ptr(lse), _ptr(split_out), _ptr(task_map), _ptr(q), _ptr(kcache), _ptr(vcache),
        _ptr(block_ids), _ptr(num_seq_kvcache), _ptr(qscale), _ptr(kscale), _ptr(vscale),
        _ptr(split_flag),
        int(bool(new_kv_included)), splitk, 0, 1, int(quant_type),
        num_batch, num_seq_q, num_head_q, num_head_k, num_head_v, num_dim_qk, num_dim_v,
        num_kvcache_blocks, block_size, num_seq_max_blocks,
        qscale.stride(0), y.stride(0), q.stride(0),
        kcache.stride(0), kcache.stride(1), kcache.stride(2),
        vcache.stride(0), vcache.stride(1), vcache.stride(2),
        _stream_of(q),
    )
    return y, args, (lse, split_out, task_map)


def _attention_decode_bf16_impl(
    q, kcache, vcache, block_ids, num_seq_kvcache, mtp, new_kv_included, use_splitk,
    task_map=None, split_flag=None, output=None,
):
    """bf16 paged decode attention; validation mirrors reference src/attention/entry.cc:411-470."""
    _require(q.is_cuda, "q tensor must be cuda")
    _require(kcache.is_cuda, "kcache tensor must be cuda")
    _require(vcache.is_cuda, "vcache tensor must be cuda")
    _require(block_ids.is_cuda, "block_ids tensor must be cuda")
    _require(block_ids.is_contiguous(), "block_ids tensor must be contiguous")
    _require(num_seq_kvcache.is_contiguous(), "num_seq_kvcache tensor must be contiguous")
    _require(block_ids.dtype == torch.int32, "block_ids dtype must be int32")
    _require(num_seq_kvcache.dtype == torch.int32, "num_seq_kvcache dtype must be int32")
    _require(mtp in (0, 1, 2, 3, 4), "we only support mtp 0, 1, 2, 3, 4.")
    _require(q.dtype == torch.bfloat16 and kcache.dtype == torch.bfloat16
             and vcache.dtype == torch.bfloat16, "q, kcache and vcache must be bfloat16")

    num_batch = num_seq_kvcache.size(0)
    num_seq_q = q.size(0) // num_batch
    _require(num_seq_q == mtp + 1, "every request num_seq_q must be mtp + 1")
    num_head_q = q.size(1)
    num_dim_qk = q.size(2)
    _require(num_dim_qk == 128, "we only support head dim 128.")
    num_kvcache_blocks = kcache.size(0)
    block_size = kcache.size(1)
    _require(block_size in (16, 32, 64), "kvcache paged blocksize must be 16, 32 or 64.")
    num_head_k = kcache.size(2)
    num_head_v = vcache.size(2)
    num_dim_v = vcache.size(3)
    num_seq_max_blocks = block_ids.size(1)
    heads_per_group = num_head_q // num_head_k
    _require(heads_per_group in (4, 8), "we only support num_head_q / num_head_k == 4 or 8.")
    _require(heads_per_group * num_seq_q <= 32,
             "heads_per_group * num_seq_q must be <= 32 (mtp 4 needs heads_per_group 4)")
    _require(q.stride(2) == 1 and q.stride(1) == num_dim_qk, "q must be contiguous in (head, dim)")
    _require(kcache.stride(3) == 1 and vcache.stride(3) == 1, "kv cache innermost dim must be contiguous")

    y = _decode_output(output, q, num_batch * num_seq_q, num_head_q)

    num_total_ctas = _num_total_ctas(q.device)
    if task_map is None:
        # task-map driven kernel: without a caller-provided map the schedule is made on the device
        # right here (the reference's static split-k path, src/attention/entry.cc:540-570)
        task_map = get_attention_decode_task_workspace(
            num_batch, int(num_seq_max_blocks) * block_size + num_seq_q, num_head_k,
            min_process_len=512, device=q.device)
        _assign_task_cuda(num_seq_kvcache, num_head_k, num_seq_q, new_kv_included, 512, task_map)
    else:
        _require(bool(use_splitk), "attention_decode_bf16: splitk must be true with a task_map.")

    splitk = num_total_ctas
    pad_heads_per_group = (heads_per_group + 7) // 8 * 8
    lse = torch.empty((num_batch, splitk, num_head_k, num_seq_q, pad_heads_per_group),
                      dtype=torch.float32, device=q.device)
    split_out = torch.empty((num_batch, splitk, num_seq_q, num_head_q, num_dim_v),
                            dtype=torch.float32, device=q.device)
    _check_rc(_lib.hpc_attention_decode_bf16_async(
        _ptr(y), _ptr(lse), _ptr(split_out), _ptr(task_map), _ptr(q), _ptr(kcache), _ptr(vcache),
        _ptr(block_ids), _ptr(num_seq_kvcache), _ptr(split_flag),
        int(bool(new_kv_included)), splitk,
        num_batch, num_seq_q, num_head_q, num_head_k, num_head_v, num_dim_qk, num_dim_v,
        num_kvcache_blocks, block_size, num_seq_max_blocks, y.stride(0), q.stride(0),
        kcache.stride(0), kcache.stride(1), kcache.stride(2),
        vcache.stride(0), vcache.stride(1), vcache.stride(2),
        _stream_of(q)), "attention_decode_bf16")
    return y


_MLA_DQK = 576
_MLA_DV = 512
_MLA_HEADS = (8, 16, 32, 64, 128)


def mla_num_query_tiles(num_head_q: int, mtp: int) -> int:
    """T = ceil(H * (mtp + 1) / 64): the 64-row query tiles of one request, the `num_head_kv` an
    MLA decode task map is built with."""
    return (num_head_q * (mtp + 1) + 63) // 64


def _mla_workspace_floats(num_total_ctas: int) -> int:
    # split-chunk partials [2C, 64, 512] and LSEs [2C, 64], the rotated walk's carry [C, 256*128+512]
    return 2 * num_total_ctas * 64 * (_MLA_DV + 1) + num_total_ctas * (256 * 128 + 512)


def _attention_decode_mla_bf16_impl(q, kv_cache, block_ids, num_seq_kvcache, softmax_scale, mtp,
                                    new_kv_included, task_map=None, output=None):
    who = "attention_decode_mla_bf16"
    _require(q.is_cuda and kv_cache.is_cuda and block_ids.is_cuda and num_seq_kvcache.is_cuda,
             f"{who}: q, kv_cache, block_ids and num_seq_kvcache must be cuda tensors")
    _require(q.dtype == torch.bfloat16 and kv_cache.dtype == torch.bfloat16,
             f"{who}: q and kv_cache must be bfloat16")
    _require(block_ids.dtype == torch.int32 and block_ids.dim() == 2 and block_ids.is_contiguous(),
             f"{who}: block_ids must be contiguous int32 [num_batch, max_blocks]")
    _require(num_seq_kvcache.dtype == torch.int32 and num_seq_kvcache.dim() == 1
             and num_seq_kvcache.is_contiguous(), f"{who}: num_seq_kvcache must be contiguous int32 [B]")
    _require(mtp in (0, 1, 2, 3), f"{who}: mtp must be 0, 1, 2 or 3")
    num_batch = num_seq_kvcache.size(0)
    _require(1 <= num_batch <= 2048, f"{who}: batch must be 1..2048")
    _require(block_ids.size(0) == num_batch, f"{who}: block_ids must have num_batch rows")
    num_seq_q = mtp + 1
    _require(q.dim() == 3 and q.size(0) == num_batch * num_seq_q,
             f"{who}: q must be [num_batch * (mtp + 1), H, 576]")
    num_head_q = q.size(1)
    _require(num_head_q in _MLA_HEADS, f"{who}: num heads must be one of {_MLA_HEADS}")
    _require(q.size(2) == _MLA_DQK, f"{who}: q head dim must be 576")
    _require(q.stride(2) == 1 and q.stride(1) == _MLA_DQK,
             f"{who}: q must be contiguous in (head, dim)")
    _require(kv_cache.dim() == 3 and kv_cache.size(2) == _MLA_DQK and kv_cache.stride(2) == 1,
             f"{who}: kv_cache must be [num_blocks, 64, 576] with contiguous rows")
    _require(kv_cache.size(1) == 64, f"{who}: page size must be 64")
    y = output
    rows = num_batch * num_seq_q
    if y is None:
        y = torch.empty((rows, num_head_q, _MLA_DV), dtype=torch.bfloat16, device=q.device)
    else:
        _require(y.is_cuda and y.device == q.device and y.dtype == torch.bfloat16,
                 f"{who}: output must be bfloat16 on q's device")
        _require(tuple(y.shape) == (rows, num_head_q, _MLA_DV),
                 f"{who}: output must have shape [num_batch * (mtp + 1), H, 512]")
        _require(y.stride(2) == 1 and y.stride(1) == _MLA_DV
                 and (rows == 1 or y.stride(0) >= num_head_q * _MLA_DV),
                 f"{who}: output rows must be [H, 512] contiguous and must not overlap")
        _require(y.data_ptr() % 16 == 0 and (rows == 1 or y.stride(0) % 8 == 0),
                 f"{who}: output and its row stride must be 16-byte aligned")
    num_tiles = mla_num_query_tiles(num_head_q, mtp)
    if task_map is None:
        task_map = get_attention_decode_task_workspace(
            num_batch, int(block_ids.size(1)) * 64 + num_seq_q, num_tiles, min_process_len=512,
            device=q.device)
        _assign_task_cuda(num_seq_kvcache, num_tiles, num_seq_q, new_kv_included, 512, task_map)
    num_total_ctas = _num_total_ctas(q.device)
    ws = torch.empty(_mla_workspace_floats(num_total_ctas), dtype=torch.float32, device=q.device)
    chunk_base = torch.empty(num_batch * num_tiles, dtype=torch.int32, device=q.device)
    _check_rc(_lib.hpc_attention_decode_mla_bf16_async(
        _ptr(y), _ptr(ws), _ptr(chunk_base), _ptr(task_map), _ptr(q), _ptr(kv_cache),
        _ptr(block_ids), num_batch, num_seq_q, num_head_q, q.size(2), kv_cache.size(0),
        kv_cache.size(1), block_ids.size(1), y.stride(0), q.stride(0), kv_cache.stride(0),
        kv_cache.stride(1), float(softmax_scale), num_total_ctas, _stream_of(q)), who)
    return y


def _assign_task_cpu(num_seq_kvcache, num_head_kv, num_seq_q, new_kv_included, min_process_len,
                     placeholder=None, num_total_ctas: _Optional[int] = None):
    """CPU scheduler -> packed host task map int8 [rows, 48] (reference entry.cc:727-778)."""
    _require(num_seq_kvcache.device.type == "cpu", "num_seq_kvcache tensor must be cpu")
    lens = num_seq_kvcache.to(torch.int32).contiguous()
    num_batch = lens.size(0)
    if num_total_ctas is None:
        num_total_ctas = _num_total_ctas()
    a = (lens.data_ptr(), num_total_ctas, num_batch, num_head_kv, num_seq_q, _TILE_N,
         int(bool(new_kv_included)), min_process_len)
    nbytes = _lib.hpc_assign_attention_decode_task_host_bytes(*a)
    _require(nbytes > 0, "assign_attention_decode_task: bad geometry")
    out = torch.zeros((nbytes // _TASK_BYTES, _TASK_BYTES), dtype=torch.int8)
    _check_rc(_lib.hpc_assign_attention_decode_task_sync(*a, out.data_ptr(), nbytes),
          "assign_attention_decode_task (cpu)")
    return out


def _assign_task_cuda(num_seq_kvcache, num_head_kv, num_seq_q, new_kv_included, min_process_len,
                      task_map):
    _require(num_seq_kvcache.is_cuda, "num_seq_kvcache tensor must be cuda")
    _require(task_map is not None, "assign_attention_decode_task_cuda must use task_map output.")
    _require(num_seq_kvcache.dtype == torch.int32 and num_seq_kvcache.is_contiguous(),
             "num_seq_kvcache must be contiguous int32")
    num_batch = num_seq_kvcache.size(0)
    _require(num_batch <= 2048, "assign_attention_decode_task_cuda only support batch_size <= 2048")
    _check_rc(_lib.hpc_assign_attention_decode_task_async(
        _ptr(task_map), _ptr(num_seq_kvcache), _num_total_ctas(num_seq_kvcache.device), num_batch,
        num_head_kv, num_seq_q, _TILE_N, int(bool(new_kv_included)), min_process_len,
        _stream_of(num_seq_kvcache)), "assign_attention_decode_task (cuda)")
    return task_map


def _blocksparse_prefill_impl(q, kcache, vcache, qscale, kscale, vscale, cu_seqlens_q, block_ids,
                              seqlens_kvcache, max_seqlens_q, quant_type, block_mask, output):
    # validation follows reference src/attention/entry.cc:266-409
    for t, name in ((q, "q"), (kcache, "kcache"), (vcache, "vcache"), (qscale, "qscale"),
                    (cu_seqlens_q, "cu_seqlens_q"), (block_ids, "block_ids"),
                    (seqlens_kvcache, "seqlens_kvcache")):
        _require(t.is_cuda, f"{name} tensor must be cuda")
    _require(q.dtype == torch.float8_e4m3fn, "q dtype must be fp8_e4m3fn")
    _require(kcache.element_size() == 1 and vcache.element_size() == 1, "kv cache must be fp8")
    _require(qscale.dtype == torch.float32 and qscale.is_contiguous(), "qscale must be contiguous float32")
    _require(cu_seqlens_q.dtype == torch.int32 and block_ids.dtype == torch.int32
             and seqlens_kvcache.dtype == torch.int32, "index tensors must be int32")
    _require(block_ids.is_contiguous(), "block_ids tensor must be contiguous")
    _require(quant_type in (0, 1), "blocksparse prefill supports quant_type 0 and 1")
    total_seq, num_head_q, dim = q.shape
    _require(dim == 128, "we only support head dim 128.")
    _require(q.stride(2) == 1 and q.stride(1) == dim, "q must be contiguous in (head, dim)")
    num_blocks, block_size, num_head_kv = kcache.size(0), kcache.size(1), kcache.size(2)
    _require(128 % block_size == 0, "128 must be divisible by the kv block size")
    _require(kcache.stride(3) == 1 and vcache.stride(3) == 1, "kv cache innermost dim must be contiguous")
    num_batch = seqlens_kvcache.size(0)
    _require(cu_seqlens_q.numel() == num_batch + 1, "cu_seqlens_q must have num_batch + 1 entries")
    _require(qscale.dim() == 3 and qscale.size(0) == num_batch and qscale.size(1) == num_head_q,
             "qscale shape must be [num_batch, num_head_q, max_seq_q_pad]")
    mask_ptr, mask_mq, mask_kb = None, 0, 0
    if block_mask is not None:
        _require(block_mask.is_cuda and block_mask.is_contiguous() and block_mask.dtype == torch.uint8,
                 "block_mask must be a contiguous cuda uint8 tensor")
        _require(block_mask.dim() == 4 and block_mask.size(0) == num_batch
                 and block_mask.size(1) == num_head_q
                 and block_mask.size(2) >= (max_seqlens_q + 127) // 128,
                 "block_mask shape must be [num_batch, num_head_q, ceil(max_seq_q/128), num_kv_tiles]")
        mask_ptr, mask_mq, mask_kb = block_mask.data_ptr(), block_mask.size(2), block_mask.size(3)
    if output is not None:
        _require(output.dtype == torch.bfloat16 and output.is_cuda
                 and tuple(output.shape) == (total_seq, num_head_q, dim) and output.stride(2) == 1
                 and output.stride(1) == dim, "output must be bf16 [total_seq, num_head_q, 128]")
        y = output
    else:
        y = torch.empty((total_seq, num_head_q, dim), dtype=torch.bfloat16, device=q.device)
    common = (
        _ptr(y), _ptr(q), _ptr(kcache), _ptr(vcache), _ptr(qscale), None, _ptr(vscale),
        _ptr(cu_seqlens_q), _ptr(block_ids), _ptr(seqlens_kvcache), mask_ptr, num_batch, total_seq,
        int(max_seqlens_q), num_head_q, num_head_kv, dim, num_blocks, block_size, block_ids.size(1),
        qscale.size(2), mask_mq, mask_kb, y.stride(0), q.stride(0), kcache.stride(0),
        kcache.stride(1), kcache.stride(2), vcache.stride(0), vcache.stride(1), vcache.stride(2))
    if quant_type == 1:
        _require(kscale.dtype == torch.float32 and vscale.dtype == torch.float32, "scales must be float32")
        args = common[:5] + (_ptr(kscale),) + common[6:] + (_stream_of(q),)
        _check_rc(_lib.hpc_attention_blocksparse_prefill_qpertoken_perhead_kvpertensor_fp8_async(*args),
                  "attention_with_kvcache_blocksparse_prefill_fp8")
    else:
        ks = kscale if kscale.dtype == torch.float32 else kscale.view(torch.float32)
        _require(ks.dim() == 4 and ks.size(0) == num_blocks and ks.size(1) == block_size // 32
                 and ks.size(2) == num_head_kv and ks.size(3) == 32 and ks.stride(3) == 1,
                 "per-token kscale must be f32 [num_blocks, block_size/32, num_head_kv, 32]")
        _require(vscale.dtype == torch.float32 and vscale.numel() == num_head_kv,
                 "per-head vscale must be f32 [num_head_kv]")
        # the stride of a size-1 dim is never applied, and torch may report any value for it
        # (1 for a contiguous [blocks, 2, 1, 32]); the kernel needs 16-byte multiples
        kst = tuple(ks.stride(i) if ks.size(i) > 1 else 0 for i in range(3))
        args = common[:5] + (_ptr(ks),) + common[6:] + kst + (_stream_of(q),)
        _check_rc(_lib.hpc_attention_blocksparse_prefill_qkpertoken_perhead_vperhead_fp8_async(*args),
                  "attention_with_kvcache_blocksparse_prefill_fp8")
    return y


_ops.define(
    "attention_with_kvcache_blocksparse_prefill_fp8(Tensor q, Tensor kcache, Tensor vcache,"
    "Tensor qscale, Tensor kscale, Tensor vscale, Tensor cu_seqlens_q,"
    "Tensor block_ids, Tensor num_seq_kvcache, int max_seqlens_q, int quant_type,"
    "Tensor? block_mask, Tensor? output) -> (Tensor)")
_ops.impl("attention_with_kvcache_blocksparse_prefill_fp8", _blocksparse_prefill_impl, "CUDA")

def _dense_prefill_fp8_impl(q, kcache, vcache, qscale, kscale, vscale, cu_seqlens_q, block_ids,
                            seqlens_kvcache, max_seqlens_q, quant_type, output):
    # reference src/attention/entry.cc:152-264: the dense path is the block-sparse kernel without
    # a mask (the reference itself instantiates it with kHasMask=false, hpc/attention.py:270-271)
    return _blocksparse_prefill_impl(q, kcache, vcache, qscale, kscale, vscale, cu_seqlens_q,
                                     block_ids, seqlens_kvcache, max_seqlens_q, quant_type, None,
                                     output)


_ops.define(
    "attention_with_kvcache_prefill_fp8(Tensor q, Tensor kcache, Tensor vcache,"
    "Tensor qscale, Tensor kscale, Tensor vscale, Tensor cu_seqlens_q,"
    "Tensor block_ids, Tensor num_seq_kvcache, int max_seqlens_q, int quant_type,"
    "Tensor? output) -> (Tensor)")
_ops.impl("attention_with_kvcache_prefill_fp8", _dense_prefill_fp8_impl, "CUDA")

def _bf16_prefill_common(who, q, output, index_tensors):
    """Checks shared by the two bf16 prefill ops; returns (total_seq, num_head_q, y)."""
    _require(q.is_cuda, "q tensor must be cuda")
    for t, name in index_tensors:
        _require(t.is_cuda, f"{name} tensor must be cuda")
        _require(t.dtype == torch.int32 and t.is_contiguous(), f"{name} must be contiguous int32")
    _require(q.dtype == torch.bfloat16, "q dtype must be bfloat16")
    _require(q.dim() == 3 and q.size(2) == 128, f"{who}: head dim must be 128")
    _require(q.stride(2) == 1 and q.stride(1) == 128, "q must be contiguous in (head, dim)")
    total_seq, num_head_q = q.size(0), q.size(1)
    if output is not None:
        _require(output.is_cuda and output.device == q.device, "output tensor must be cuda, on q's device")
        _require(output.dtype == torch.bfloat16, "output dtype must be bfloat16")
        _require(output.is_contiguous(), "output tensor must be contiguous")
        _require(tuple(output.shape) == (total_seq, num_head_q, 128),
                 "output must have shape [total_seq_q, num_head_q, 128]")
        y = output
    else:
        y = torch.empty((total_seq, num_head_q, 128), dtype=torch.bfloat16, device=q.device)
    return total_seq, num_head_q, y


def _attention_prefill_bf16_impl(q, k, v, seqlens_q, cu_seqlens_q, max_seqlens_q, output=None):
    """Varlen causal self-attention on contiguous bf16 q/k/v; validation follows reference
    src/attention/entry.cc:15-70."""
    who = "attention_prefill_bf16"
    total_seq, num_head_q, y = _bf16_prefill_common(
        who, q, output, ((seqlens_q, "seqlens_q"), (cu_seqlens_q, "cu_seqlens_q")))
    _require(k.is_cuda and v.is_cuda, "k and v tensors must be cuda")
    _require(k.dtype == torch.bfloat16 and v.dtype == torch.bfloat16, "k and v dtype must be bfloat16")
    _require(k.dim() == 3 and v.dim() == 3 and k.size(2) == 128 and v.size(2) == 128,
             f"{who}: head dim must be 128")
    _require(k.size(0) == total_seq and v.size(0) == total_seq and k.size(1) == v.size(1),
             "k and v must be [total_seq_q, num_head_kv, 128]")
    _require(k.stride(2) == 1 and k.stride(1) == 128 and v.stride(2) == 1 and v.stride(1) == 128,
             "k and v must be contiguous in (head, dim)")
    num_head_kv = k.size(1)
    _require(num_head_kv > 0 and num_head_q % num_head_kv == 0,
             "num_head_q must be a multiple of num_head_kv")
    num_batch = seqlens_q.size(0)
    _require(cu_seqlens_q.numel() == num_batch + 1, "cu_seqlens_q must have num_batch + 1 entries")
    _check_rc(_lib.hpc_attention_prefill_bf16_async(
        _ptr(y), _ptr(q), _ptr(k), _ptr(v), _ptr(seqlens_q), _ptr(cu_seqlens_q), num_batch,
        total_seq, int(max_seqlens_q), 128, 128, num_head_q, num_head_kv, y.stride(0), q.stride(0),
        k.stride(0), v.stride(0), _stream_of(q)), who)
    return y


def _attention_with_kvcache_prefill_bf16_impl(q, kcache, vcache, cu_seqlens_q, block_ids,
                                              seqlens_kvcache, max_seqlens_q, output=None):
    """Causal (chunked) prefill over the paged bf16 KV cache; validation follows reference
    src/attention/entry.cc:72-150."""
    who = "attention_with_kvcache_prefill_bf16"
    total_seq, num_head_q, y = _bf16_prefill_common(
        who, q, output, ((cu_seqlens_q, "cu_seqlens_q"), (block_ids, "block_ids"),
                         (seqlens_kvcache, "seqlens_kvcache")))
    _require(kcache.is_cuda and vcache.is_cuda, "kv cache tensors must be cuda")
    _require(kcache.dtype == torch.bfloat16 and vcache.dtype == torch.bfloat16,
             "kcache and vcache dtype must be bfloat16")
    _require(kcache.dim() == 4 and kcache.shape == vcache.shape,
             "kcache and vcache must both be [num_blocks, block_size, num_head_kv, 128]")
    _require(kcache.size(3) == 128, f"{who}: head dim must be 128")
    _require(kcache.stride(3) == 1 and vcache.stride(3) == 1, "kv cache innermost dim must be contiguous")
    num_blocks, block_size, num_head_kv = kcache.size(0), kcache.size(1), kcache.size(2)
    _require(block_size in (16, 32, 64), "kvcache paged blocksize must be 16, 32 or 64.")
    _require(num_head_q % num_head_kv == 0, "num_head_q must be a multiple of num_head_kv")
    num_batch = cu_seqlens_q.numel() - 1
    _require(num_batch > 0 and seqlens_kvcache.numel() == num_batch
             and block_ids.dim() == 2 and block_ids.size(0) == num_batch,
             "cu_seqlens_q [B+1], seqlens_kvcache [B] and block_ids [B, max_blocks] disagree on B")
    _check_rc(_lib.hpc_attention_with_kvcache_prefill_bf16_async(
        _ptr(y), _ptr(q), _ptr(kcache), _ptr(vcache), _ptr(cu_seqlens_q), _ptr(block_ids),
        _ptr(seqlens_kvcache), num_batch, total_seq, int(max_seqlens_q), 128, 128, num_head_q,
        num_head_kv, num_blocks, block_size, block_ids.size(1), y.stride(0), q.stride(0),
        kcache.stride(0), kcache.stride(1), kcache.stride(2),
        vcache.stride(0), vcache.stride(1), vcache.stride(2), _stream_of(q)), who)
    return y


_MLA_PREFILL_DQK = 192
_MLA_PREFILL_DV = 128
_MLA_PREFILL_DPE = 64


def _attention_prefill_mla_bf16_impl(q, k_nope, k_pe, v, cu_seqlens_q, cu_seqlens_kv,
                                     max_seqlen_q, softmax_scale, output=None):
    who = "attention_prefill_mla_bf16"
    for t, name in ((q, "q"), (k_nope, "k_nope"), (k_pe, "k_pe"), (v, "v")):
        _require(t.dtype == torch.bfloat16, f"{who}: {name} must be bfloat16")
    for t, name in ((cu_seqlens_q, "cu_seqlens_q"), (cu_seqlens_kv, "cu_seqlens_kv")):
        _require(t.dtype == torch.int32 and t.dim() == 1 and t.is_contiguous(),
                 f"{who}: {name} must be contiguous int32 [num_batch + 1]")
    num_batch = cu_seqlens_q.numel() - 1
    _require(num_batch >= 1 and cu_seqlens_kv.numel() == num_batch + 1,
             f"{who}: cu_seqlens_q and cu_seqlens_kv must both have num_batch + 1 >= 2 entries")
    _require(q.dim() == 3 and q.size(2) == _MLA_PREFILL_DQK, f"{who}: q must be [total_q, H, 192]")
    total_q, num_head = q.size(0), q.size(1)
    _require(1 <= num_head <= 128, f"{who}: num heads must be 1..128")
    _require(q.stride(2) == 1 and (num_head == 1 or q.stride(1) == _MLA_PREFILL_DQK),
             f"{who}: q must be contiguous in (head, dim)")
    _require(k_nope.dim() == 3 and tuple(k_nope.shape[1:]) == (num_head, _MLA_PREFILL_DV),
             f"{who}: k_nope must be [total_kv, H, 128]")
    _require(v.dim() == 3 and tuple(v.shape[1:]) == (num_head, _MLA_PREFILL_DV),
             f"{who}: v must be [total_kv, H, 128]")
    _require(k_pe.dim() == 2 and k_pe.size(1) == _MLA_PREFILL_DPE, f"{who}: k_pe must be [total_kv, 64]")
    total_kv = k_nope.size(0)
    _require(total_kv >= 1 and v.size(0) == total_kv and k_pe.size(0) == total_kv,
             f"{who}: k_nope, k_pe and v must hold the same total_kv >= 1 tokens")
    _require(k_nope.stride(2) == 1 and v.stride(2) == 1 and k_pe.stride(1) == 1,
             f"{who}: k_nope, k_pe and v rows must be contiguous")
    for t, name in ((q, "q"), (k_nope, "k_nope"), (k_pe, "k_pe"), (v, "v"),
                    (cu_seqlens_q, "cu_seqlens_q"), (cu_seqlens_kv, "cu_seqlens_kv")):
        _require(t.is_cuda and t.device == q.device, f"{who}: {name} must be a cuda tensor on q's device")
    y = output
    if y is None:
        y = torch.empty((total_q, num_head, _MLA_PREFILL_DV), dtype=torch.bfloat16, device=q.device)
    else:
        _require(y.is_cuda and y.device == q.device and y.dtype == torch.bfloat16,
                 f"{who}: output must be bfloat16 on q's device")
        _require(y.is_contiguous() and tuple(y.shape) == (total_q, num_head, _MLA_PREFILL_DV),
                 f"{who}: output must be contiguous [total_q, H, 128]")

    def st(t, i, unit):
        # the stride of a size-1 dim is never applied, and torch may report any value for it
        return t.stride(i) if t.size(i) > 1 else unit

    _check_rc(_lib.hpc_attention_prefill_mla_bf16_async(
        _ptr(y), _ptr(q), _ptr(k_nope), _ptr(k_pe), _ptr(v), _ptr(cu_seqlens_q), _ptr(cu_seqlens_kv),
        num_batch, total_q, total_kv, int(max_seqlen_q), num_head, q.size(2), v.size(2),
        num_head * _MLA_PREFILL_DV, st(q, 0, num_head * _MLA_PREFILL_DQK),
        st(k_nope, 0, num_head * _MLA_PREFILL_DV), st(k_nope, 1, _MLA_PREFILL_DV),
        st(k_pe, 0, _MLA_PREFILL_DPE), st(v, 0, num_head * _MLA_PREFILL_DV), st(v, 1, _MLA_PREFILL_DV),
        float(softmax_scale), _stream_of(q)), who)
    return y


# schemas of reference src/attention/entry.cc (attention_prefill_bf16,
# attention_with_kvcache_prefill_bf16 registrations)
_ops.define(
    "attention_prefill_bf16(Tensor q, Tensor k, Tensor v, Tensor seqlens_q, Tensor cu_seqlens_q, "
    "int max_seqlens_q, Tensor? output) -> (Tensor)")
_ops.impl("attention_prefill_bf16", _attention_prefill_bf16_impl, "CUDA")

_ops.define(
    "attention_with_kvcache_prefill_bf16(Tensor q, Tensor kcache, Tensor vcache,"
    "Tensor cu_seqlens_q, Tensor block_ids, Tensor num_seq_kvcache, int max_seqlens_q, "
    "Tensor? output) -> (Tensor)")
_ops.impl("attention_with_kvcache_prefill_bf16", _attention_with_kvcache_prefill_bf16_impl, "CUDA")

_ops.define(
    "attention_prefill_mla_bf16(Tensor q, Tensor k_nope, Tensor k_pe, Tensor v, "
    "Tensor cu_seqlens_q, Tensor cu_seqlens_kv, int max_seqlen_q, float softmax_scale, "
    "Tensor? output) -> (Tensor)")
_ops.impl("attention_prefill_mla_bf16", _attention_prefill_mla_bf16_impl, "CUDA")

_ops.define(
    "attention_decode_bf16(Tensor q, Tensor! kcache, Tensor! vcache, Tensor block_ids, Tensor "
    "num_seq_kvcache, int mtp, bool new_kv_included, bool use_splitk, Tensor? task_map, "
    "Tensor? split_flag, Tensor? output) -> "
    "(Tensor)")
_ops.impl("attention_decode_bf16", _attention_decode_bf16_impl, "CUDA")

_ops.define(
    "attention_decode_mla_bf16(Tensor q, Tensor kv_cache, Tensor block_ids, Tensor num_seq_kvcache, "
    "float softmax_scale, int mtp, bool new_kv_included, Tensor? task_map, Tensor? output) -> "
    "(Tensor)")
_ops.impl("attention_decode_mla_bf16", _attention_decode_mla_bf16_impl, "CUDA")

_ops.define(
    "attention_decode_fp8(Tensor q, Tensor! kcache, Tensor! vcache, Tensor block_ids, Tensor "
    "num_seq_kvcache, Tensor qscale, Tensor kscale, Tensor vscale, int mtp, bool "
    "new_kv_included, int quant_type, bool "
    "use_splitk, Tensor? task_map, Tensor? split_flag, Tensor? output) -> (Tensor)")
_ops.impl("attention_decode_fp8", _attention_decode_fp8_impl, "CUDA")

_ops.define(
    "assign_attention_decode_task(Tensor num_seq_kvcache, int num_head_kv, int num_seq_q, bool "
    "new_kv_included, int min_process_len, Tensor? task_map) -> (Tensor)")
_ops.impl("assign_attention_decode_task", _assign_task_cpu, "CPU")
_ops.impl("assign_attention_decode_task", _assign_task_cuda, "CUDA")


# --------------------------------------------------------------------------------------------
# public API (signatures of reference hpc/attention.py)
# --------------------------------------------------------------------------------------------
def attention_with_kvcache_prefill_fp8(
    q: Tensor,
    kcache: Tensor,
    vcache: Tensor,
    qscale: Tensor,
    kscale: Tensor,
    vscale: Tensor,
    cu_seqlens_q: Tensor,
    block_ids: Tensor,
    seqlens_kvcache: Tensor,
    max_seqlens_q: int,
    quant_type: QuantType = QuantType.QPERTOKEN_PERHEAD_KPERTENSOR_VPERTENSOR,
    output: Tensor = None,
) -> Tensor:
    """Dense causal prefill over the paged FP8 KV cache (contract of reference
    hpc/attention.py:148-250): the last `seqlens_q[b]` tokens of each request attend to all
    `seqlens_kvcache[b]` cached tokens causally. Same tensors as
    `attention_with_kvcache_blocksparse_prefill_fp8` without a block mask; both quant schemes."""
    return torch.ops.hpc.attention_with_kvcache_prefill_fp8(
        q, kcache, vcache, qscale, kscale, vscale, cu_seqlens_q, block_ids, seqlens_kvcache,
        max_seqlens_q, quant_type.value, output)


def attention_with_kvcache_blocksparse_prefill_fp8(
    q: Tensor,
    kcache: Tensor,
    vcache: Tensor,
    qscale: Tensor,
    kscale: Tensor,
    vscale: Tensor,
    cu_seqlens_q: Tensor,
    block_ids: Tensor,
    seqlens_kvcache: Tensor,
    max_seqlens_q: int,
    quant_type: QuantType = QuantType.QPERTOKEN_PERHEAD_KPERTENSOR_VPERTENSOR,
    block_mask: _Optional[Tensor] = None,
    output: Tensor = None,
) -> Tensor:
    """Unified dense / block-sparse causal prefill over the paged FP8 KV cache
    (contract of reference hpc/attention.py:253-338).

      q [total_seq, Hq, 128] e4m3; caches [blocks, 64, Hkv, 128] e4m3 (NHD or HND via strides);
      qscale f32 [B, Hq, max_seq_q_pad]; cu_seqlens_q [B+1]; block_ids [B, max_blocks];
      seqlens_kvcache [B] = total kv tokens (incl. the new ones);
      block_mask u8 [B, Hq, ceil(max_seq_q/128), Kb] (absolute 128-key tile index; 1 = compute) or
      None for dense. quant_type 1: kscale/vscale [1]; quant_type 0: kscale f32
      [blocks, 2, Hkv, 32] (may be passed viewed as fp8), vscale [Hkv].
    Returns bf16 [total_seq, Hq, 128]. A Q tile with no active KV tile yields NaN rows, as in the
    reference."""
    return torch.ops.hpc.attention_with_kvcache_blocksparse_prefill_fp8(
        q, kcache, vcache, qscale, kscale, vscale, cu_seqlens_q, block_ids, seqlens_kvcache,
        max_seqlens_q, quant_type.value, block_mask, output)


def attention_prefill_bf16(
    q: Tensor,
    k: Tensor,
    v: Tensor,
    seqlens_q: Tensor,
    cu_seqlens_q: Tensor,
    max_seqlens_q: int,
    output: Tensor = None,
) -> Tensor:
    """Varlen causal self-attention in bf16 (contract of reference hpc/attention.py:15-64):
    softmax(Q K^T / sqrt(128)) V per request, query i seeing keys 0..i of its own request.

      q           [total_seq, num_head_q, 128] bfloat16, contiguous in (head, dim)
      k, v        [total_seq, num_head_kv, 128] bfloat16, same; num_head_q % num_head_kv == 0
      seqlens_q   [num_batch] int32, equal to the lengths cu_seqlens_q gives
      cu_seqlens_q [num_batch + 1] int32: request b is rows cu_seqlens_q[b] .. cu_seqlens_q[b+1]-1
      max_seqlens_q  at least the longest request (a larger value only costs idle work items)
      output      optional contiguous bf16 [total_seq, num_head_q, 128]
    Returns bf16 [total_seq, num_head_q, 128]."""
    return torch.ops.hpc.attention_prefill_bf16(q, k, v, seqlens_q, cu_seqlens_q, max_seqlens_q,
                                                output)


def attention_with_kvcache_prefill_bf16(
    q: Tensor,
    kcache: Tensor,
    vcache: Tensor,
    cu_seqlens_q: Tensor,
    block_ids: Tensor,
    seqlens_kvcache: Tensor,
    max_seqlens_q: int,
    output: Tensor = None,
) -> Tensor:
    """Causal prefill, including chunked prefill, over the paged bf16 KV cache (contract of
    reference hpc/attention.py:67-145): the `sq` new tokens of request b are the last ones of its
    `skv = seqlens_kvcache[b]` cached tokens, and new token i sees cached keys j <= skv - sq + i.

      q           [total_seq, num_head_q, 128] bfloat16, contiguous in (head, dim)
      kcache, vcache [num_blocks, block_size, num_head_kv, 128] bfloat16, block_size 16 / 32 / 64,
                  any strides on dims 0-2 (NHD or HND). Slots past skv in a request's last page are
                  never read into the result, whatever they hold.
      cu_seqlens_q [num_batch + 1] int32; block_ids [num_batch, max_blocks] int32;
      seqlens_kvcache [num_batch] int32 (cached tokens including the new ones)
      output      optional contiguous bf16 [total_seq, num_head_q, 128]
    Returns bf16 [total_seq, num_head_q, 128]. Requests with sq = 0 write nothing."""
    return torch.ops.hpc.attention_with_kvcache_prefill_bf16(
        q, kcache, vcache, cu_seqlens_q, block_ids, seqlens_kvcache, max_seqlens_q, output)


def attention_prefill_mla_bf16(
    q: Tensor,
    k_nope: Tensor,
    k_pe: Tensor,
    v: Tensor,
    cu_seqlens_q: Tensor,
    cu_seqlens_kv: Tensor,
    max_seqlen_q: int,
    softmax_scale: float,
    output: Tensor = None,
) -> Tensor:
    """Multi-head latent attention (MLA) prefill in the un-absorbed form, varlen and causal.

      q           [total_q, H, 192] bfloat16: per head q_nope (128) then the RoPE'd q_pe (64);
                  contiguous in (head, dim), token stride a multiple of 8 elements. 1 <= H <= 128.
      k_nope, v   [total_kv, H, 128] bfloat16, e.g. kv[..., :128] and kv[..., 128:] of a
                  kv_b_proj output [total_kv, H, 256]
      k_pe        [total_kv, 64] bfloat16, the RoPE'd key all heads share, e.g. latent[:, 512:] of
                  a [total_kv, 576] latent buffer
                  (k_nope, v and k_pe: any token and head strides that are multiples of 8
                  elements, contiguous rows, 16-byte aligned; no copy is made)
      cu_seqlens_q, cu_seqlens_kv  [B + 1] int32: request b has nq = cu_seqlens_q[b+1] -
                  cu_seqlens_q[b] queries and nk = cu_seqlens_kv[b+1] - cu_seqlens_kv[b] keys
      max_seqlen_q  at least the longest nq (a larger value only costs idle work items)
      softmax_scale  used as given: s = (q_nope . k_nope + q_pe . k_pe) * softmax_scale
                  (DeepSeek-V3: mscale^2 / sqrt(192))
      output      optional contiguous bf16 [total_q, H, 128]
    Causal masking is bottom-right: query i of request b sees its keys j <= nk - nq + i. So
    cu_seqlens_kv == cu_seqlens_q is causal self-attention, and nk > nq is chunked prefill over a
    prefix. Returns bf16 [total_q, H, 128]; a query that sees no key (nk < nq) gets zeros, and
    rows of requests with nq = 0 are not written. The launch never synchronises, so it can be
    captured in a CUDA graph."""
    return torch.ops.hpc.attention_prefill_mla_bf16(
        q, k_nope, k_pe, v, cu_seqlens_q, cu_seqlens_kv, max_seqlen_q, float(softmax_scale), output)


def attention_decode_bf16(
    q: Tensor,
    kcache: Tensor,
    vcache: Tensor,
    block_ids: Tensor,
    num_seq_kvcache: Tensor,
    mtp: int = 0,
    new_kv_included: bool = False,
    splitk: bool = True,
    task_map: Tensor = None,
    split_flag: Tensor = None,
    output: Tensor = None,
) -> Tensor:
    """BF16 paged decode attention: softmax(Q K^T / sqrt(d)) V with the MTP causal tail.

    Same contract as reference hpc/attention.py:341-417.
      q          [num_batch * num_seq_q, num_head_q, 128] bfloat16 (num_seq_q = mtp + 1)
      kcache     [num_blocks, block_size, num_head_kv, 128] bfloat16, block_size 16 / 32 / 64, any
                 strides on dims 0-2 (NHD or HND); unused slots of a request's last block zero
      vcache     same
      block_ids  [num_batch, max_blocks] int32;  num_seq_kvcache [num_batch] int32
      task_map   from get_attention_decode_task_workspace + assign_attention_decode_task (None:
                 scheduled on the device inside the call)
    Returns bf16 [num_batch * num_seq_q, num_head_q, 128].
    """
    return torch.ops.hpc.attention_decode_bf16(
        q, kcache, vcache, block_ids, num_seq_kvcache, mtp, new_kv_included, splitk, task_map,
        split_flag, output,
    )


def attention_decode_mla_bf16(
    q: Tensor,
    kv_cache: Tensor,
    block_ids: Tensor,
    num_seq_kvcache: Tensor,
    softmax_scale: float,
    mtp: int = 0,
    new_kv_included: bool = False,
    task_map: Tensor = None,
    output: Tensor = None,
) -> Tensor:
    """Absorbed multi-head latent attention (MLA) decode over a paged bf16 latent cache.

      q           [B * (mtp + 1), H, 576] bfloat16, contiguous in (head, dim); each head is
                  [q_nope . W_UK (512) | q_pe after RoPE (64)]. H in {8, 16, 32, 64, 128}.
      kv_cache    [num_blocks, 64, 576] bfloat16; each row is [kv_c (512) | k_pe after RoPE (64)].
                  Rows must be contiguous; the token and block strides may be any multiple of 8
                  elements (a view into a wider allocation works). Slots past a request's last
                  token never reach the output, whatever they hold (NaN included).
      block_ids   [B, max_blocks] int32;  num_seq_kvcache [B] int32, B <= 2048
      softmax_scale  used as given: s = (q . k) * softmax_scale (DeepSeek-V3: mscale^2 / sqrt(192))
      mtp         0..3; MTP row sq of a request with n keys sees keys <= n - (mtp + 1) + sq, where n
                  is num_seq_kvcache[b] (+ mtp + 1 unless new_kv_included), as attention_decode_bf16
      task_map    from get_attention_decode_task_workspace + assign_attention_decode_task built with
                  num_head_kv = T = mla_num_query_tiles(H, mtp) = ceil(H (mtp + 1) / 64), the
                  64-row query tiles of a request (None: scheduled on the device inside the call)
      output      optional bf16 [B * (mtp + 1), H, 512]; rows may be strided (16-byte aligned)
    Returns y = softmax(s) . kv_cache[..., :512], bf16 [B * (mtp + 1), H, 512]. The launch
    allocates nothing outside torch's allocator and never synchronises, so it can be captured in a
    CUDA graph (with a pre-assigned task map)."""
    return torch.ops.hpc.attention_decode_mla_bf16(
        q, kv_cache, block_ids, num_seq_kvcache, float(softmax_scale), mtp, new_kv_included,
        task_map, output)


def attention_decode_fp8(
    q: Tensor,
    kcache: Tensor,
    vcache: Tensor,
    block_ids: Tensor,
    num_seq_kvcache: Tensor,
    qscale: Tensor,
    kscale: Tensor,
    vscale: Tensor,
    mtp: int = 0,
    new_kv_included: bool = False,
    quant_type: QuantType = QuantType.QPERTOKEN_PERHEAD_KPERTENSOR_VPERTENSOR,
    splitk: bool = True,
    task_map: Tensor = None,
    split_flag: Tensor = None,
    output: Tensor = None,
) -> Tensor:
    """FP8 paged decode attention: softmax(Q K^T * qscale * kscale / sqrt(d)) V * vscale.

    Same contract as reference hpc/attention.py:420-517.
      q          [num_batch * num_seq_q, num_head_q, 128] float8_e4m3fn
      kcache     [num_blocks, 64, num_head_kv, 128] float8_e4m3fn, any strides on dims 0-2
      vcache     same; unused slots of a request's last block must be zero
      block_ids  [num_batch, max_blocks] int32;  num_seq_kvcache [num_batch] int32
      qscale     [num_batch * num_seq_q, num_head_q] f32
      kscale, vscale  quant_type 1: [1] f32 each; quant_type 0: kscale = the cache allocation's
                 scale rows (f32 [num_blocks, 2, num_head_kv, 32], same strides as kcache),
                 vscale [num_head_kv] f32
      task_map   from get_attention_decode_task_workspace + assign_attention_decode_task
    Returns bf16 [num_batch * num_seq_q, num_head_q, 128].
    """
    return torch.ops.hpc.attention_decode_fp8(
        q, kcache, vcache, block_ids, num_seq_kvcache, qscale, kscale, vscale, mtp,
        new_kv_included, quant_type.value, splitk, task_map, split_flag, output,
    )


def get_attention_decode_task_workspace(
    max_num_batch: int, max_seqlen: int, num_head_kv: int, min_process_len: int = 512, device=None
):
    """Allocate (and zero) the decode task map; sizing identical to reference
    hpc/attention.py:520-582 (worst case over 64-key tiles and 1..4 CTAs per SM), so a workspace
    is interchangeable between builds.

    Returns int8 [task_map_byte_size] on `device` (default: the current CUDA device) with header
    ints [2]=num_head_kv, [3]=max_num_batch, [4]=sched bytes. (`device` is an extension over the
    reference signature: the attention entry passes q.device.)
    """
    kTaskInfoByteSize = _TASK_BYTES
    kMaxCtaPerSm = 4
    num_sm_count = _ffi.sm_count(device)
    max_num_cta_count = num_sm_count * kMaxCtaPerSm

    kMinTileN = 64
    total_tiles = max_num_batch * num_head_kv * ((max_seqlen + kMinTileN - 1) // kMinTileN)
    max_num_tasks = 0
    for cta_per_sm in (4, 3, 2, 1):
        num_ctas = num_sm_count * cta_per_sm
        tile_per_cta = max((total_tiles + num_ctas - 1) // num_ctas, min_process_len // kMinTileN)
        max_num_tasks = max(max_num_tasks, (tile_per_cta + 1) * num_ctas + 1)

    int_size = 4
    num_chunks_bytes = max_num_batch * num_head_kv * int_size
    max_num_batch_pad = (
        (num_chunks_bytes + kTaskInfoByteSize - 1) // kTaskInfoByteSize * kTaskInfoByteSize
    )
    num_cta_count_pad = (max_num_cta_count + _TASK_INTS - 1) // _TASK_INTS * _TASK_INTS * int_size

    sched_need_byte_size = max_num_tasks * kTaskInfoByteSize + max_num_batch_pad
    workspace_byte_size = sched_need_byte_size + 2 * num_cta_count_pad
    # Zeroed workspace with the three header ints the scheduler reads, built without a host
    # synchronisation: a per-(device, geometry) device-resident template is cloned (device-to-device,
    # stream-ordered, legal under CUDA-graph capture once the template exists).
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    key = (dev.index if dev.index is not None else torch.cuda.current_device(), workspace_byte_size,
           num_head_kv, max_num_batch, sched_need_byte_size)
    tmpl = _WORKSPACE_TEMPLATES.get(key)
    if tmpl is None:
        tmpl = torch.zeros(workspace_byte_size, dtype=torch.int8, device=dev)
        header = torch.tensor([0, 0, num_head_kv, max_num_batch, sched_need_byte_size], dtype=torch.int32)
        tmpl.view(torch.int32)[:5].copy_(header)
        if len(_WORKSPACE_TEMPLATES) > 64:
            _WORKSPACE_TEMPLATES.clear()
        _WORKSPACE_TEMPLATES[key] = tmpl
    return tmpl.clone()


def assign_attention_decode_task(
    num_seq_kvcache: Tensor,
    task_map: Tensor,
    num_head_kv: int,
    mtp: int,
    new_kv_included: bool,
    min_process_len: int = 512,
) -> Tensor:
    """Populate a task map (reference hpc/attention.py:585-626).

    `num_seq_kvcache` on CPU -> host scheduler + splice into the device workspace;
    on CUDA -> device scheduler. Both produce identical bytes. (`mtp` carries num_seq_q,
    as in the reference's tests.)
    """
    if num_seq_kvcache.device.type == "cpu":
        host = torch.ops.hpc.assign_attention_decode_task(
            num_seq_kvcache, num_head_kv, mtp, new_kv_included, min_process_len, None
        ).reshape(-1)
        task_map[:8].copy_(host[:8], non_blocking=True)
        task_map[20:24].copy_(host[20:24], non_blocking=True)
        task_map[48 : host.numel()].copy_(host[48:], non_blocking=True)
        # header int 6 (a pad word in the reference): tiles per kv head, as the device scheduler
        # writes it; the decode kernels rotate their bin walk by it (csrc/decode_common.cuh)
        ns = num_seq_kvcache.to(torch.int64) + (0 if new_kv_included else int(mtp))
        tiles = int(((ns + _TILE_N - 1) // _TILE_N).sum())
        task_map[24:28].copy_(torch.tensor([tiles], dtype=torch.int32).view(torch.int8))
        return task_map
    return torch.ops.hpc.assign_attention_decode_task(
        num_seq_kvcache, num_head_kv, mtp, new_kv_included, min_process_len, task_map
    )


def print_attention_decode_task(task_map: Tensor) -> None:
    """Pretty-print a task map (same fields as reference hpc/attention.py:629-696)."""
    task = task_map.view(torch.int32).reshape(-1)
    task = task[: task.numel() // _TASK_INTS * _TASK_INTS].reshape(-1, _TASK_INTS).cpu()
    ntpc1 = int(task[0][0])
    num_total_ctas = int(task[0][1])
    num_head_kv = int(task[0][2])
    max_num_batch = int(task[0][3])
    chunk_row = 1 + num_total_ctas * ntpc1
    chunks = task[chunk_row:].reshape(-1)[: num_head_kv * max_num_batch]
    print(f"\n[decode task map] num_tile_per_cta={ntpc1 - 1}, num_head_kv={num_head_kv}, "
          f"max_num_batch={max_num_batch}, num_total_ctas={num_total_ctas}, "
          f"max_num_chunks={int(task[0][5])}")
    print(f"num_chunks[ihead_kv, ibatch]:\n{chunks.reshape(num_head_kv, max_num_batch)}\n")
    gid = 0
    empty = 0
    for icta in range(num_total_ctas):
        start = 1 + icta * ntpc1
        if int(task[start][0]) < 0:
            empty += 1
            continue
        print(f"#######CTA{icta}########")
        for i in range(ntpc1 - 1):
            r = task[start + i].tolist()
            if r[0] < 0 or r[1] < 0:
                break
            print(f"task:{gid}, ihead_kv:{r[0]}, ibatch:{r[1]}, ichunk:{r[2]}, iseq_start:{r[3]}, "
                  f"num_seqkv:{r[4]}, num_seqkvcache:{r[5]}, num_tile_kv:{r[6]}, "
                  f"num_tile_full:{r[7]}, is_casual_chunk:{r[8]}")
            gid += 1
    print(f"[idle] {empty}/{num_total_ctas} bins were empty")


@torch.library.register_fake("hpc::attention_with_kvcache_blocksparse_prefill_fp8")
def _blocksparse_prefill_fake(q, kcache, vcache, qscale, kscale, vscale, cu_seqlens_q, block_ids,
                              num_seq_kvcache, max_seqlens_q, quant_type, block_mask, output):
    if output is not None:
        return output
    return torch.empty((q.size(0), q.size(1), vcache.size(3)), dtype=torch.bfloat16, device=q.device)


@torch.library.register_fake("hpc::attention_with_kvcache_prefill_fp8")
def _dense_prefill_fp8_fake(q, kcache, vcache, qscale, kscale, vscale, cu_seqlens_q, block_ids,
                            num_seq_kvcache, max_seqlens_q, quant_type, output):
    if output is not None:
        return output
    return torch.empty((q.size(0), q.size(1), vcache.size(3)), dtype=torch.bfloat16, device=q.device)


@torch.library.register_fake("hpc::attention_decode_bf16")
def _attention_decode_bf16_fake(
    q, kcache, vcache, block_ids, num_seq_kvcache, mtp, new_kv_included, use_splitk,
    task_map=None, split_flag=None, output=None,
):
    if output is not None:
        return output
    return torch.empty_like(q)


@torch.library.register_fake("hpc::attention_decode_mla_bf16")
def _attention_decode_mla_bf16_fake(q, kv_cache, block_ids, num_seq_kvcache, softmax_scale, mtp,
                                    new_kv_included, task_map=None, output=None):
    if output is not None:
        return output
    return q.new_empty((q.size(0), q.size(1), _MLA_DV))


@torch.library.register_fake("hpc::attention_decode_fp8")
def _attention_decode_fp8_fake(
    q, kcache, vcache, block_ids, num_seq_kvcache, qscale, kscale, vscale, mtp, new_kv_included,
    quant_type, use_splitk, task_map, split_flag, output,
):
    if output is not None:
        return output
    return torch.empty((q.size(0), q.size(1), vcache.size(3)), dtype=torch.bfloat16,
                       device=q.device)


@torch.library.register_fake("hpc::attention_prefill_bf16")
def _attention_prefill_bf16_fake(q, k, v, seqlens_q, cu_seqlens_q, max_seqlens_q, output=None):
    if output is not None:
        return output
    return torch.empty((q.size(0), q.size(1), v.size(2)), dtype=torch.bfloat16, device=q.device)


@torch.library.register_fake("hpc::attention_with_kvcache_prefill_bf16")
def _attention_with_kvcache_prefill_bf16_fake(q, kcache, vcache, cu_seqlens_q, block_ids,
                                              num_seq_kvcache, max_seqlens_q, output=None):
    if output is not None:
        return output
    return torch.empty((q.size(0), q.size(1), vcache.size(3)), dtype=torch.bfloat16,
                       device=q.device)


@torch.library.register_fake("hpc::attention_prefill_mla_bf16")
def _attention_prefill_mla_bf16_fake(q, k_nope, k_pe, v, cu_seqlens_q, cu_seqlens_kv, max_seqlen_q,
                                     softmax_scale, output=None):
    if output is not None:
        return output
    return q.new_empty((q.size(0), q.size(1), _MLA_PREFILL_DV))
