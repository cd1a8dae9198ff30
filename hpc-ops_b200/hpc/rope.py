"""RoPE + optional QK RMSNorm + paged KV-cache store (API of reference hpc/rope.py:8-232)."""
from typing import Optional as _Optional, Tuple as _Tuple

import torch
from torch import Tensor

from . import _ops
from ._ffi import (check as _check_rc, lib as _lib, ptr as _ptr, require as _require,
                   stream_of as _stream_of)

_FP8_MAX = 448.0


def _geometry(kcache, vcache, qkv, num_seqlen_per_req, kvcache_indices):
    # reference src/rope/entry.cc:30-44
    num_req = num_seqlen_per_req.size(0)
    num_rows = qkv.size(0)
    num_kv_heads, qk_head_dim = kcache.size(2), kcache.size(3)
    v_head_dim = vcache.size(3)
    num_q_heads = (qkv.size(1) - num_kv_heads * qk_head_dim - num_kv_heads * v_head_dim) // qk_head_dim
    _require(num_q_heads > 0 and
             qkv.size(1) == num_q_heads * qk_head_dim + num_kv_heads * (qk_head_dim + v_head_dim),
             "qkv row length does not match the cache head geometry")
    for t, name in ((kcache, "kcache"), (vcache, "vcache")):
        _require(t.stride(3) == 1 and t.stride(2) == t.size(3) and t.stride(1) == t.size(2) * t.size(3),
                 f"{name} pages must be contiguous [block_size, num_kv_heads, head_dim]")
    return (num_req, num_rows, num_q_heads, num_kv_heads, qk_head_dim, v_head_dim, kcache.size(1),
            kvcache_indices.size(1))


def _common_checks(qkv, cos_sin, num_seqlen_per_req, q_index, kvcache_indices, qk_norm_policy,
                   q_norm_weight, k_norm_weight):
    for t, name in ((qkv, "qkv"), (cos_sin, "cos_sin"), (num_seqlen_per_req, "num_seqlen_per_req"),
                    (kvcache_indices, "kvcache_indices"), (q_index, "q_index")):
        _require(t.is_cuda and t.is_contiguous(), f"{name} tensor must be a contiguous cuda tensor")
    _require(qkv.dtype == torch.bfloat16, "qkv must be bfloat16")
    _require(cos_sin.dtype == torch.float32, "cos_sin must be float32")
    _require(num_seqlen_per_req.dtype == torch.int32 and q_index.dtype == torch.int32
             and kvcache_indices.dtype == torch.int32, "index tensors must be int32")
    _require(0 <= qk_norm_policy <= 2, "qk_norm_policy must be 0, 1 or 2")
    if qk_norm_policy != 0:
        _require(q_norm_weight is not None and k_norm_weight is not None
                 and q_norm_weight.dtype == torch.float32 and k_norm_weight.dtype == torch.float32,
                 "q/k norm weights (float32) are required when qk_norm_policy != 0")


def _rope_impl(kcache, vcache, qkv, cos_sin, num_seqlen_per_req, q_index, kvcache_indices,
               is_prefill, q_norm_weight=None, k_norm_weight=None, out_q=None, out_k=None, out_v=None,
               qk_norm_policy=0):
    # (trailing arguments equal to their schema defaults are not passed to a Python kernel)
    # reference src/rope/entry.cc:16-92
    _common_checks(qkv, cos_sin, num_seqlen_per_req, q_index, kvcache_indices, qk_norm_policy,
                   q_norm_weight, k_norm_weight)
    _require(kcache.dtype == torch.bfloat16 and vcache.dtype == torch.bfloat16, "kv caches must be bfloat16")
    (num_req, num_rows, hq, hkv, dqk, dv, block_size, max_blocks) = _geometry(
        kcache, vcache, qkv, num_seqlen_per_req, kvcache_indices)
    if out_q is None:
        out_q = torch.empty((num_rows, hq, dqk), dtype=qkv.dtype, device=qkv.device)
    for t, name in ((out_q, "out_q"), (out_k, "out_k"), (out_v, "out_v")):
        _require(t is None or (t.is_contiguous() and t.dtype == torch.bfloat16), f"{name} must be contiguous bf16")
    _check_rc(_lib.hpc_rope_norm_store_kv_async(
        _ptr(out_q), _ptr(kcache), _ptr(vcache), _ptr(out_k), _ptr(out_v), _ptr(qkv), _ptr(cos_sin),
        _ptr(num_seqlen_per_req), _ptr(q_index), _ptr(kvcache_indices), _ptr(q_norm_weight),
        _ptr(k_norm_weight), kcache.stride(0), vcache.stride(0), num_req, max_blocks, block_size,
        num_rows, hq, hkv, dqk, dv, int(bool(is_prefill)), int(qk_norm_policy), _stream_of(qkv)),
        "rope_norm_store_kv")
    return out_q


def _rope_fp8_impl(kcache, vcache, qkv, cos_sin, num_seqlen_per_req, q_index, kvcache_indices,
                   is_prefill, k_scale, v_scale, quant_policy, max_seqlens, upper_max, q_scale_inv,
                   q_norm_weight, k_norm_weight, out_q, out_k, out_v, qk_norm_policy):
    # reference src/rope/entry.cc:94-219
    _common_checks(qkv, cos_sin, num_seqlen_per_req, q_index, kvcache_indices, qk_norm_policy,
                   q_norm_weight, k_norm_weight)
    _require(k_scale.dim() == 1 and k_scale.size(0) == 1, "k_scale must contain 1 element")
    _require(v_scale.dim() == 1 and v_scale.size(0) == 1, "v_scale must contain 1 element")
    _require(quant_policy in (1, 2), "quant_policy must be 1 or 2")
    _require(kcache.element_size() == 1 and vcache.element_size() == 1, "kv caches must be 1-byte dtype")
    (num_req, num_rows, hq, hkv, dqk, dv, block_size, max_blocks) = _geometry(
        kcache, vcache, qkv, num_seqlen_per_req, kvcache_indices)
    um = _FP8_MAX
    if upper_max is not None:
        _require(not (float(upper_max) > _FP8_MAX), "upper_max should not be larger than fp8_max")
        um = float(upper_max)
    if out_q is None:
        out_q = torch.empty((num_rows, hq, dqk), dtype=torch.float8_e4m3fn, device=qkv.device)
    for t, name in ((out_q, "out_q"), (out_k, "out_k"), (out_v, "out_v")):
        _require(t is None or (t.is_contiguous() and t.dtype == torch.float8_e4m3fn),
                 f"{name} must be contiguous float8_e4m3fn")
    q_scale = None
    if quant_policy == 1:
        if is_prefill:
            pad128 = (int(max_seqlens) + 127) // 128 * 128
            q_scale = torch.empty((num_req, hq, pad128), dtype=torch.float32, device=qkv.device)
        else:
            q_scale = torch.empty((num_rows, hq), dtype=torch.float32, device=qkv.device)
    else:
        _require(q_scale_inv is not None and q_scale_inv.dtype == torch.float32,
                 "q_scale_inv required for quant_policy=2")
    split_k_flag = torch.empty((num_req, hkv), dtype=torch.int32, device=qkv.device)
    _check_rc(_lib.hpc_rope_norm_store_kv_fp8_async(
        _ptr(out_q), _ptr(kcache), _ptr(vcache), _ptr(out_k), _ptr(out_v), _ptr(split_k_flag),
        _ptr(q_scale), _ptr(qkv), _ptr(cos_sin), _ptr(num_seqlen_per_req), _ptr(q_index),
        _ptr(kvcache_indices), _ptr(q_norm_weight), _ptr(k_norm_weight), _ptr(k_scale), _ptr(v_scale),
        _ptr(q_scale_inv), um, int(max_seqlens), kcache.stride(0), vcache.stride(0), num_req,
        max_blocks, block_size, num_rows, hq, hkv, dqk, dv, int(bool(is_prefill)),
        int(qk_norm_policy), int(quant_policy), _stream_of(qkv)), "rope_norm_store_kv_fp8")
    return out_q, q_scale, split_k_flag


_ops.define(
    "rope_norm_store_kv(Tensor! kcache, Tensor! vcache, Tensor qkv, Tensor cos_sin, "
    "Tensor num_seqlen_per_req, Tensor q_index, Tensor kvcache_indices, bool is_prefill, "
    "Tensor? q_norm_weight, Tensor? k_norm_weight, "
    "Tensor? out_q=None, Tensor? out_k=None, Tensor? out_v=None, int qk_norm_policy=0) -> "
    "Tensor")
_ops.impl("rope_norm_store_kv", _rope_impl, "CUDA")


def rope_norm_store_kv(
    key_cache: Tensor, value_cache: Tensor, qkv: Tensor, cos_sin: Tensor, num_seqlen_per_req: Tensor,
    q_index: Tensor, kvcache_indices: Tensor, is_prefill: bool,
    q_norm_weight: _Optional[Tensor] = None, k_norm_weight: _Optional[Tensor] = None,
    out_q: _Optional[Tensor] = None, out_k: _Optional[Tensor] = None, out_v: _Optional[Tensor] = None,
    qk_norm_policy: int = 0,
) -> Tensor:
    """NeoX RoPE on Q/K of the packed bf16 `qkv` rows, optional per-head RMSNorm (policy 1: after,
    2: before the rotation), K/V written into the paged bf16 cache (or into out_k / out_v), the
    unused tail of each request's last page zeroed. Returns the rotated Q [rows, Hq, D]
    (contract of reference hpc/rope.py:8-105).

    The call writes only the slots of its rows and, for a request with rows in the call, the
    tail of the page of its last token. A request with no new rows leaves its pages untouched,
    and with out_k / out_v given no cache byte is written at all (no tail is zeroed either)."""
    return torch.ops.hpc.rope_norm_store_kv(
        key_cache, value_cache, qkv, cos_sin, num_seqlen_per_req, q_index, kvcache_indices,
        is_prefill, q_norm_weight, k_norm_weight, out_q, out_k, out_v, qk_norm_policy)


@torch.library.register_fake("hpc::rope_norm_store_kv")
def _rope_fake(kcache, vcache, qkv, cos_sin, num_seqlen_per_req, q_index, kvcache_indices, is_prefill,
               q_norm_weight=None, k_norm_weight=None, out_q=None, out_k=None, out_v=None,
               qk_norm_policy=0):
    hkv, dqk, dv = kcache.shape[-2], kcache.shape[-1], vcache.shape[-1]
    hq = (qkv.shape[-1] - hkv * dqk - hkv * dv) // dqk
    return torch.empty(qkv.shape[0], hq, dqk, dtype=qkv.dtype, device=qkv.device)


# The reference returns an empty tensor for q_scale under quant_policy 2 and its Python test accepts
# None (tests/test_rope.py:349); torch custom ops cannot return None inside a tuple, so the FP8 entry
# point is a plain function here (the bf16 one above is a registered op with the reference schema).
def rope_norm_store_kv_fp8(
    key_cache: Tensor, value_cache: Tensor, qkv: Tensor, cos_sin: Tensor, num_seqlen_per_req: Tensor,
    q_index: Tensor, kvcache_indices: Tensor, is_prefill: bool, k_scale: Tensor, v_scale: Tensor,
    quant_policy: int, max_seqlens: int = 0, upper_max: _Optional[float] = None,
    q_scale_inv: _Optional[Tensor] = None, q_norm_weight: _Optional[Tensor] = None,
    k_norm_weight: _Optional[Tensor] = None, out_q: _Optional[Tensor] = None,
    out_k: _Optional[Tensor] = None, out_v: _Optional[Tensor] = None, qk_norm_policy: int = 0,
) -> _Tuple[Tensor, _Optional[Tensor], Tensor]:
    """FP8 variant (contract of reference hpc/rope.py:108-232): K and V are stored as e4m3 with the
    static per-tensor scales (x / scale); Q is quantised per token and head with a dynamic scale
    amax / upper_max (quant_policy 1; scales returned as [num_req, Hq, pad128(max_seqlens)] in
    prefill and [rows, Hq] in decode) or with the caller's q_scale_inv (quant_policy 2, q_scale is
    None). Returns (q_fp8, q_scale, split_k_flag[num_req, Hkv] zeroed, also when there are no
    rows). Cache writes follow rope_norm_store_kv: only the rows' slots and the last page's tail
    of a request with rows; nothing with out_k / out_v."""
    return _rope_fp8_impl(key_cache, value_cache, qkv, cos_sin, num_seqlen_per_req, q_index,
                          kvcache_indices, is_prefill, k_scale, v_scale, int(quant_policy),
                          int(max_seqlens), upper_max, q_scale_inv, q_norm_weight, k_norm_weight,
                          out_q, out_k, out_v, int(qk_norm_policy))
