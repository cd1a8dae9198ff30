"""Stem block-mask generation (API of reference hpc/stem.py): the four stages that score a paged FP8
KV cache against packed FP8 queries at 128-token block granularity and keep each query block's top
key blocks, giving the `block_mask` of `attention_with_kvcache_blocksparse_prefill_fp8`.

    mask = hpc.stem_paged_kv(q, kcache, vcache, qscale, kscale, vscale, block_ids, cu_seqlens_q,
                             seqlens_kvcache, num_prompt_tokens)
    out = hpc.attention_with_kvcache_blocksparse_prefill_fp8(..., block_mask=mask)

The prep ops size their outputs from the longest request (`.max().item()`, a host synchronisation);
`stem_oam_gemm` and `stem_tpd` never synchronise and can be captured in a CUDA graph."""
from typing import Tuple

import torch
from torch import Tensor

from . import _ops
from ._ffi import (check as _check_rc, lib as _lib, ptr as _ptr, require as _require,
                   stream_of as _stream_of)
from .attention import QuantType

_BLOCK = 128
_STRIDE = 16
_MAX_KB = 32768


def _check_geometry(who: str, stem_block_size: int, stem_stride: int):
    _require(stem_block_size == _BLOCK and stem_stride == _STRIDE,
             f"{who}: only stem_block_size=128, stem_stride=16 is supported "
             f"(got {stem_block_size}, {stem_stride})")


def _check_lens(who: str, name: str, t: Tensor, n: int, device):
    _require(t.device == device and t.dtype == torch.int32 and t.dim() == 1 and t.shape[0] == n
             and t.is_contiguous(), f"{who}: {name} must be a contiguous int32 [{n}] tensor on {device}")


def _prep_paged_kv_impl(kcache, vcache, kscale, vscale, kv_indices, kv_seq_lens, lambda_mag,
                        stem_block_size, stem_stride, quant_type):
    who = "stem_oam_prep_paged_kv"
    dev = kcache.device
    _require(quant_type in (0, 1), f"{who}: quant_type only support 0/1 (got {quant_type})")
    _check_geometry(who, stem_block_size, stem_stride)
    _require(kcache.dim() == 4 and vcache.dim() == 4 and kcache.shape == vcache.shape,
             f"{who}: kcache and vcache must both be [num_blocks, block_size, num_kv_heads, 128]")
    _require(kcache.dtype == torch.float8_e4m3fn and vcache.dtype == torch.float8_e4m3fn,
             f"{who}: kcache and vcache must be float8_e4m3fn")
    num_blocks, block_size, hkv, dim_qk = kcache.shape
    _require(block_size in (32, 64), f"{who}: kv_block_size must be 32 or 64, got {block_size}")
    _require(dim_qk == 128 and vcache.shape[3] == 128,
             f"{who}: unsupported dim_qk={dim_qk} dim_v={vcache.shape[3]} (expected 128, 128)")
    _require(kcache.stride(3) == 1 and vcache.stride(3) == 1, f"{who}: the head dim must be contiguous")
    _require(kv_indices.dtype == torch.int32 and kv_indices.dim() == 2 and kv_indices.stride(1) == 1
             and kv_indices.stride(0) == kv_indices.shape[1],
             f"{who}: kv_indices must be a contiguous int32 [num_batch, max_blocks_per_req] tensor")
    B = kv_seq_lens.shape[0] if kv_seq_lens.dim() == 1 else -1
    _require(kv_indices.shape[0] == B, f"{who}: kv_indices has {kv_indices.shape[0]} rows for {B} requests")
    _check_lens(who, "kv_seq_lens", kv_seq_lens, B, dev)
    _require(kscale.dtype.itemsize in (1, 4), f"{who}: kscale dtype must be float or fp8")
    if quant_type == 1:
        _require(kscale.dtype == torch.float32 and kscale.numel() >= 1 and vscale.dtype == torch.float32
                 and vscale.numel() >= 1, f"{who}: quant_type 1 takes fp32 kscale [1] and vscale [1]")
    else:
        esz = kscale.dtype.itemsize
        _require(kscale.dim() == 4 and kscale.shape[0] == num_blocks and kscale.shape[2] == hkv
                 and kscale.shape[3] * esz == 128 and kscale.stride(3) == 1
                 and all(kscale.stride(i) * esz % 4 == 0 for i in range(3)),
                 f"{who}: quant_type 0 takes kscale [num_blocks, block_size / 32, num_kv_heads, 32] fp32 "
                 "(or its fp8 view)")
        _require(vscale.dtype == torch.float32 and vscale.numel() >= hkv and vscale.is_contiguous(),
                 f"{who}: quant_type 0 takes fp32 vscale [num_kv_heads]")
    max_kv = int(kv_seq_lens.max().item()) if B > 0 else 0
    _require(max_kv <= kv_indices.shape[1] * block_size,
             f"{who}: kv_seq_lens up to {max_kv} exceed the block table's "
             f"{kv_indices.shape[1]} x {block_size} tokens")
    max_kb = (max_kv + _BLOCK - 1) // _BLOCK
    max_down = max_kb * (_BLOCK // _STRIDE)
    _require(kcache.is_cuda and vcache.device == dev and kscale.device == dev and vscale.device == dev
             and kv_indices.device == dev and kv_seq_lens.device == dev,
             f"{who}: all tensors must be CUDA tensors on one device")
    kflat = torch.empty(B, hkv, max_kb, _STRIDE * 128, dtype=torch.bfloat16, device=dev)
    vbias = torch.empty(B, hkv, max_kb, dtype=torch.float32, device=dev)
    v_norm_down = torch.empty(B, hkv, max_down, dtype=torch.float32, device=dev)
    stream = _stream_of(kcache)
    ks, vs = kcache.stride(), vcache.stride()
    if quant_type == 1:
        rc = _lib.hpc_stem_oam_prep_paged_kv_qpertoken_perhead_kvpertensor_dim128_async(
            _ptr(kflat), _ptr(vbias), _ptr(kcache), _ptr(vcache), _ptr(kscale), _ptr(vscale),
            _ptr(kv_indices), _ptr(kv_seq_lens), B, 128, 128, hkv, num_blocks, block_size,
            kv_indices.shape[1], stem_block_size, stem_stride, float(lambda_mag), max_kb, max_down,
            ks[0], vs[0], ks[1], ks[2], vs[1], vs[2], _ptr(v_norm_down), stream)
    else:
        esz = kscale.dtype.itemsize
        kss = [kscale.stride(i) * esz // 4 for i in range(3)]
        rc = _lib.hpc_stem_oam_prep_paged_kv_qkpertoken_perhead_vperhead_dim128_async(
            _ptr(kflat), _ptr(vbias), _ptr(kcache), _ptr(vcache), _ptr(kscale), _ptr(vscale),
            _ptr(kv_indices), _ptr(kv_seq_lens), B, 128, 128, hkv, num_blocks, block_size,
            kscale.shape[1], kv_indices.shape[1], stem_block_size, stem_stride, float(lambda_mag),
            max_kb, max_down, ks[0], vs[0], kss[0], kss[1], kss[2], ks[1], ks[2], vs[1], vs[2],
            _ptr(v_norm_down), stream)
    _check_rc(rc, who)
    return kflat, vbias


def _prep_varlen_q_impl(q_fp8, qscale, q_seq_lens, cu_seqlens_q, stem_block_size, stem_stride):
    who = "stem_oam_prep_varlen_q"
    dev = q_fp8.device
    _require(q_fp8.is_contiguous(), f"{who}: q_fp8 must be contiguous")
    _check_geometry(who, stem_block_size, stem_stride)
    _require(q_fp8.dim() == 3 and q_fp8.dtype == torch.float8_e4m3fn,
             f"{who}: q_fp8 must be float8_e4m3fn [total_tokens, num_q_heads, 128]")
    _require(q_fp8.shape[2] == 128, f"{who}: expected dim_qk=128, got {q_fp8.shape[2]}")
    hq = q_fp8.shape[1]
    B = q_seq_lens.shape[0] if q_seq_lens.dim() == 1 else -1
    _check_lens(who, "q_seq_lens", q_seq_lens, B, dev)
    _check_lens(who, "cu_seqlens_q", cu_seqlens_q, B + 1, dev)
    _require(qscale.dim() == 3, f"{who}: qscale must be [B, Hq, max_q_pad]")
    _require(qscale.dtype == torch.float32 and qscale.shape[0] == B and qscale.shape[1] == hq,
             f"{who}: qscale must be fp32 [{B}, {hq}, max_q_pad]")
    max_q = int(q_seq_lens.max().item()) if B > 0 else 0
    _require(max_q <= qscale.shape[2], f"{who}: q_seq_lens up to {max_q} exceed qscale's {qscale.shape[2]}")
    max_qb = (max_q + _BLOCK - 1) // _BLOCK
    _require(q_fp8.is_cuda and qscale.device == dev and q_seq_lens.device == dev
             and cu_seqlens_q.device == dev, f"{who}: all tensors must be CUDA tensors on one device")
    qflat = torch.empty(B, hq, max_qb, _STRIDE * 128, dtype=torch.bfloat16, device=dev)
    _check_rc(_lib.hpc_stem_oam_prep_varlen_q_dim128_async(
        _ptr(qflat), _ptr(q_fp8), _ptr(qscale), _ptr(q_seq_lens), _ptr(cu_seqlens_q), B, hq,
        q_fp8.stride(0), stem_block_size, stem_stride, max_qb, qscale.stride(0), qscale.stride(1),
        qscale.stride(2), _stream_of(q_fp8)), who)
    return qflat


def _gemm_impl(qflat, kflat, vbias, q_seq_lens, kv_seq_lens, stem_block_size, stem_stride, causal):
    who = "stem_oam_gemm"
    dev = qflat.device
    _check_geometry(who, stem_block_size, stem_stride)
    _require(qflat.dim() == 4 and kflat.dim() == 4 and qflat.dtype == torch.bfloat16
             and kflat.dtype == torch.bfloat16 and qflat.is_contiguous() and kflat.is_contiguous(),
             f"{who}: qflat and kflat must be contiguous bf16 [B, H, blocks, 2048]")
    B, hq, max_qb, inner = qflat.shape
    _require(kflat.shape[0] == B, f"{who}: batch size mismatch between qflat and kflat")
    _require(kflat.shape[3] == inner, f"{who}: kFlatDim mismatch between qflat ({inner}) and kflat "
             f"({kflat.shape[3]})")
    _require(inner // stem_stride == 128 and inner % stem_stride == 0,
             f"{who}: expected dim_qk=128, got {inner / stem_stride}")
    hkv, max_kb = kflat.shape[1], kflat.shape[2]
    _require(hkv > 0 and hq % hkv == 0, f"{who}: num_head_q ({hq}) must be divisible by num_head_kv ({hkv})")
    _require(vbias.dtype == torch.float32 and vbias.is_contiguous()
             and tuple(vbias.shape) == (B, hkv, max_kb),
             f"{who}: vbias shape mismatch, expected [{B}, {hkv}, {max_kb}] fp32 contiguous")
    _check_lens(who, "q_seq_lens", q_seq_lens, B, dev)
    _check_lens(who, "kv_seq_lens", kv_seq_lens, B, dev)
    _require(qflat.is_cuda and kflat.device == dev and vbias.device == dev and q_seq_lens.device == dev
             and kv_seq_lens.device == dev, f"{who}: all tensors must be CUDA tensors on one device")
    logits = torch.empty(B, hq, max_qb, max_kb, dtype=torch.bfloat16, device=dev)
    _check_rc(_lib.hpc_stem_oam_gemm_dim128_async(
        _ptr(logits), _ptr(qflat), _ptr(kflat), _ptr(vbias), _ptr(q_seq_lens), _ptr(kv_seq_lens), B,
        hq, hkv, max_qb, max_kb, stem_block_size, stem_stride, int(bool(causal)), _stream_of(qflat)),
        who)
    return logits


def _tpd_impl(block_logits, q_seq_lens, kv_seq_lens, num_prompt_tokens, block_size, alpha,
              initial_blocks, window_size, k_block_num_rate_medium, k_block_num_bias_medium,
              k_block_num_rate_large, k_block_num_bias_large):
    who = "stem_tpd"
    dev = block_logits.device
    _require(block_logits.dtype == torch.bfloat16, "block_logits must be bfloat16")
    _require(block_logits.is_contiguous(), "block_logits must be contiguous")
    _require(block_logits.dim() == 4, f"{who}: block_logits must be [num_batch, num_heads, max_Qb, max_Kb]")
    _require(block_size == _BLOCK, f"{who}: block_size must be 128 (got {block_size})")
    B, H, max_qb, max_kb = block_logits.shape
    for name, t in (("q_seq_lens", q_seq_lens), ("kv_seq_lens", kv_seq_lens),
                    ("num_prompt_tokens", num_prompt_tokens)):
        _require(t.dtype == torch.int32, f"{name} must be int32, got {t.dtype}")
        _check_lens(who, name, t, B, dev)
    _require(max_kb <= _MAX_KB, f"stem_tpd: max_Kb={max_kb} exceeds {_MAX_KB} limit")
    _require(block_logits.is_cuda and q_seq_lens.device == dev and kv_seq_lens.device == dev
             and num_prompt_tokens.device == dev, f"{who}: all tensors must be CUDA tensors on one device")
    mask = torch.empty(B, H, max_qb, max_kb, dtype=torch.uint8, device=dev)
    _check_rc(_lib.hpc_stem_tpd_async(
        _ptr(mask), _ptr(block_logits), _ptr(q_seq_lens), _ptr(kv_seq_lens), _ptr(num_prompt_tokens),
        B, H, max_qb, max_kb, block_size, float(alpha), int(initial_blocks), int(window_size),
        float(k_block_num_rate_medium), int(k_block_num_bias_medium), float(k_block_num_rate_large),
        int(k_block_num_bias_large), _stream_of(block_logits)), who)
    return mask


_ops.define("stem_oam_prep_paged_kv(Tensor kcache, Tensor vcache, Tensor kscale, Tensor vscale, "
            "Tensor kv_indices, Tensor kv_seq_lens, float lambda_mag, int stem_block_size, "
            "int stem_stride, int quant_type) -> (Tensor, Tensor)")
_ops.impl("stem_oam_prep_paged_kv", _prep_paged_kv_impl, "CUDA")
_ops.define("stem_oam_prep_varlen_q(Tensor q_fp8, Tensor qscale, Tensor q_seq_lens, "
            "Tensor cu_seqlens_q, int stem_block_size, int stem_stride) -> Tensor")
_ops.impl("stem_oam_prep_varlen_q", _prep_varlen_q_impl, "CUDA")
_ops.define("stem_oam_gemm(Tensor qflat, Tensor kflat, Tensor vbias, Tensor q_seq_lens, "
            "Tensor kv_seq_lens, int stem_block_size, int stem_stride, bool causal) -> Tensor")
_ops.impl("stem_oam_gemm", _gemm_impl, "CUDA")
_ops.define("stem_tpd(Tensor block_logits, Tensor q_seq_lens, Tensor kv_seq_lens, "
            "Tensor num_prompt_tokens, int block_size, float alpha, int initial_blocks, "
            "int window_size, float k_block_num_rate_medium, int k_block_num_bias_medium, "
            "float k_block_num_rate_large, int k_block_num_bias_large) -> Tensor")
_ops.impl("stem_tpd", _tpd_impl, "CUDA")


@torch.library.register_fake("hpc::stem_oam_prep_paged_kv")
def _prep_paged_kv_fake(kcache, vcache, kscale, vscale, kv_indices, kv_seq_lens, lambda_mag,
                        stem_block_size, stem_stride, quant_type):
    # upper bound: every request fills its block table
    max_kb = (kv_indices.size(1) * kcache.size(1) + stem_block_size - 1) // stem_block_size
    B, hkv = kv_seq_lens.size(0), kcache.size(2)
    return (kcache.new_empty((B, hkv, max_kb, stem_stride * kcache.size(3)), dtype=torch.bfloat16),
            kcache.new_empty((B, hkv, max_kb), dtype=torch.float32))


@torch.library.register_fake("hpc::stem_oam_prep_varlen_q")
def _prep_varlen_q_fake(q_fp8, qscale, q_seq_lens, cu_seqlens_q, stem_block_size, stem_stride):
    max_qb = (qscale.size(2) + stem_block_size - 1) // stem_block_size
    return q_fp8.new_empty((q_seq_lens.size(0), q_fp8.size(1), max_qb, stem_stride * q_fp8.size(2)),
                           dtype=torch.bfloat16)


@torch.library.register_fake("hpc::stem_oam_gemm")
def _gemm_fake(qflat, kflat, vbias, q_seq_lens, kv_seq_lens, stem_block_size, stem_stride, causal):
    return qflat.new_empty((qflat.size(0), qflat.size(1), qflat.size(2), kflat.size(2)),
                           dtype=torch.bfloat16)


@torch.library.register_fake("hpc::stem_tpd")
def _tpd_fake(block_logits, q_seq_lens, kv_seq_lens, num_prompt_tokens, block_size, alpha,
              initial_blocks, window_size, k_block_num_rate_medium, k_block_num_bias_medium,
              k_block_num_rate_large, k_block_num_bias_large):
    return torch.empty_like(block_logits, dtype=torch.uint8)


def stem_oam_prep_paged_kv(
    kcache: Tensor,
    vcache: Tensor,
    kscale: Tensor,
    vscale: Tensor,
    kv_indices: Tensor,
    kv_seq_lens: Tensor,
    lambda_mag: float = 0.3,
    stem_block_size: int = 128,
    stem_stride: int = 16,
    quant_type: QuantType = QuantType.QPERTOKEN_PERHEAD_KPERTENSOR_VPERTENSOR,
) -> Tuple[Tensor, Tensor]:
    """K_flat and V_bias from the paged FP8 KV cache (first stage of the Stem pipeline).

    kcache, vcache: [num_blocks, kv_block_size (32 or 64), num_kv_heads, 128] float8_e4m3fn, NHD
    or HND (read through their strides). kscale / vscale by `quant_type`:
    QPERTOKEN_PERHEAD_KPERTENSOR_VPERTENSOR: [1] fp32 each;
    QPERTOKEN_PERHEAD_KPERTOKEN_PERHEAD_VPERHEAD: kscale [num_blocks, kv_block_size / 32,
    num_kv_heads, 32] fp32 (or an fp8 view of the same storage), vscale [num_kv_heads] fp32.
    kv_indices [num_batch, max_blocks_per_req] int32 block table, kv_seq_lens [num_batch] int32.

    Returns kflat bf16 [num_batch, num_kv_heads, max_Kb, 16 * 128]: for 128-key block kb, group g
    (0..15) is the fp32 sum of the dequantised K rows kb * 128 + g + 16 r (r < 8, rows < kv_len),
    stored in segment 15 - g; and vbias fp32 [num_batch, num_kv_heads, max_Kb]: with x the max of
    ||v * vscale|| over each 16 consecutive rows (rows past kv_len count as 0), over the request's
    ceil(kv_len / 128) * 8 values of log(x + 1e-6) with mean m and unbiased std s, vbias[kb] is the
    mean over the block's 8 values of lambda_mag * relu((log(x + 1e-6) - m) / (s + 1e-6)).
    max_Kb = ceil(max(kv_seq_lens) / 128) (a host synchronisation); blocks past a request's own
    length are left unwritten.
    """
    return torch.ops.hpc.stem_oam_prep_paged_kv(kcache, vcache, kscale, vscale, kv_indices,
                                                kv_seq_lens, lambda_mag, stem_block_size,
                                                stem_stride, QuantType(quant_type).value)


def stem_oam_prep_varlen_q(
    q_fp8: Tensor,
    qscale: Tensor,
    q_seq_lens: Tensor,
    cu_seqlens_q: Tensor,
    stem_block_size: int = 128,
    stem_stride: int = 16,
) -> Tensor:
    """Q_flat from packed FP8 Q: q_fp8 [total_tokens, num_q_heads, 128] float8_e4m3fn (contiguous),
    qscale [num_batch, num_q_heads, max_seq_q_pad] fp32 per-token scales (read through its strides),
    q_seq_lens [num_batch] and cu_seqlens_q [num_batch + 1] int32.

    Returns qflat bf16 [num_batch, num_q_heads, max_Qb, 16 * 128]: group g of query block qb is the
    fp32 sum of qscale * q over tokens qb * 128 + g + 16 r (r < 8, tokens < q_len), in natural group
    order. max_Qb = ceil(max(q_seq_lens) / 128) (a host synchronisation).
    """
    return torch.ops.hpc.stem_oam_prep_varlen_q(q_fp8, qscale, q_seq_lens, cu_seqlens_q,
                                                stem_block_size, stem_stride)


def stem_oam_gemm(
    qflat: Tensor,
    kflat: Tensor,
    vbias: Tensor,
    q_seq_lens: Tensor,
    kv_seq_lens: Tensor,
    stem_block_size: int = 128,
    stem_stride: int = 16,
    causal: bool = True,
) -> Tensor:
    """block_logits bf16 [num_batch, num_q_heads, max_Qb, max_Kb] = qflat . kflat^T / 64 +
    vbias[kv head] (fp32 accumulation; q head h reads kv head h / (Hq / Hkv)). -inf where
    qb >= ceil(q_len / 128), kb >= ceil(kv_len / 128) or, when causal,
    qb + ceil((kv_len - q_len) / 128) < kb. No host synchronisation: capturable in a CUDA graph.
    """
    return torch.ops.hpc.stem_oam_gemm(qflat, kflat, vbias, q_seq_lens, kv_seq_lens,
                                       stem_block_size, stem_stride, causal)


def stem_tpd(
    block_logits: Tensor,
    q_seq_lens: Tensor,
    kv_seq_lens: Tensor,
    num_prompt_tokens: Tensor,
    block_size: int = 128,
    alpha: float = 1.0,
    initial_blocks: int = 4,
    window_size: int = 4,
    k_block_num_rate_medium: float = 0.2,
    k_block_num_bias_medium: int = 30,
    k_block_num_rate_large: float = 0.1,
    k_block_num_bias_large: int = 30,
) -> Tensor:
    """Block mask u8 [num_batch, num_heads, max_Qb, max_Kb] (1 = compute) from block_logits bf16.

    Per row (query block q_row of a request), with P = ceil(num_prompt_tokens / 128) (pass the same
    value for every chunk of a prompt; for normal prefill pass kv_seq_lens): the budget k is P when
    P < 56, int(P * rate_medium) + bias_medium when P < 160, else int(P * rate_large) + bias_large,
    then decays linearly toward k * alpha for absolute query blocks q_pos = q_row +
    ceil((kv_len - q_len) / 128) >= k. The top-k threshold T is the largest bf16 key (order-
    preserving 16-bit map; -inf, +inf and NaN never selected) with count(key >= T) >= budget, so ties
    at T are all kept; a budget covering every finite value keeps them all. Also kept: the first
    `initial_blocks` columns, the `window_size` columns ending at the diagonal
    min(q_pos, ceil(kv_len / 128) - 1), and the diagonal. Columns and rows outside the request are 0.
    max_Kb <= 32768. No host synchronisation: capturable in a CUDA graph.
    """
    return torch.ops.hpc.stem_tpd(block_logits, q_seq_lens, kv_seq_lens, num_prompt_tokens,
                                  block_size, alpha, initial_blocks, window_size,
                                  k_block_num_rate_medium, k_block_num_bias_medium,
                                  k_block_num_rate_large, k_block_num_bias_large)


def stem_paged_kv(
    q_fp8: Tensor,
    kcache: Tensor,
    vcache: Tensor,
    qscale: Tensor,
    kscale: Tensor,
    vscale: Tensor,
    kv_indices: Tensor,
    cu_seqlens_q: Tensor,
    kv_seq_lens: Tensor,
    num_prompt_tokens: Tensor,
    lambda_mag: float = 0.3,
    alpha: float = 1.0,
    stem_block_size: int = 128,
    stem_stride: int = 16,
    causal: bool = True,
    initial_blocks: int = 4,
    window_size: int = 4,
    k_block_num_rate_medium: float = 0.2,
    k_block_num_bias_medium: int = 30,
    k_block_num_rate_large: float = 0.1,
    k_block_num_bias_large: int = 30,
    quant_type: QuantType = QuantType.QPERTOKEN_PERHEAD_KPERTENSOR_VPERTENSOR,
) -> Tensor:
    """End-to-end Stem mask for the paged FP8 KV cache: prep_paged_kv -> prep_varlen_q -> oam_gemm
    -> tpd (see each stage). q_seq_lens is derived from cu_seqlens_q. Returns the u8 mask
    [num_batch, num_q_heads, max_Qb, max_Kb] that attention_with_kvcache_blocksparse_prefill_fp8
    takes as `block_mask`."""
    q_seq_lens = (cu_seqlens_q[1:] - cu_seqlens_q[:-1]).to(torch.int32)
    kflat, vbias = stem_oam_prep_paged_kv(kcache, vcache, kscale, vscale, kv_indices, kv_seq_lens,
                                          lambda_mag, stem_block_size, stem_stride, quant_type)
    qflat = stem_oam_prep_varlen_q(q_fp8, qscale, q_seq_lens, cu_seqlens_q, stem_block_size,
                                   stem_stride)
    block_logits = stem_oam_gemm(qflat, kflat, vbias, q_seq_lens, kv_seq_lens, stem_block_size,
                                 stem_stride, causal)
    return stem_tpd(block_logits, q_seq_lens, kv_seq_lens, num_prompt_tokens, stem_block_size,
                    alpha, initial_blocks, window_size, k_block_num_rate_medium,
                    k_block_num_bias_medium, k_block_num_rate_large, k_block_num_bias_large)
