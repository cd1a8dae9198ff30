"""BF16 x FP32 route GEMM (API of reference hpc/gemm.py) and the dense blockwise FP8 GEMM of the
linear layers of a blockwise-FP8 checkpoint (no reference counterpart)."""
from typing import Optional

import torch
from torch import Tensor

from . import _ops
from ._ffi import (check as _check_rc, lib as _lib, ptr as _ptr, require as _require,
                   stream_of as _stream_of)


def _gemm_bf16xfp32_impl(x, w_high, w_low, scale, use_fp32_output, use_splitk, split_flag):
    # reference src/gemm/sm90/entry.cc:86-144
    _require(x.is_cuda and w_high.is_cuda and w_low.is_cuda, "tensors must be cuda")
    _require(x.is_contiguous(), "x tensor must be contiguous")
    _require(w_high.is_contiguous(), "w_high tensor must be contiguous")
    _require(w_low.is_contiguous(), "w_low tensor must be contiguous")
    _require(x.dtype == torch.bfloat16, "x dtype must be bfloat16")
    _require(w_high.dtype == torch.bfloat16, "w_high dtype must be bfloat16")
    _require(w_low.dtype == torch.bfloat16, "w_low dtype must be bfloat16")
    m, k = x.shape
    n = w_high.size(0)
    _require(n % 64 == 0, "n must to be divided by 64.")
    _require(tuple(w_low.shape) == tuple(w_high.shape) and w_high.size(1) == k, "weight shape mismatch")
    split_k = _lib.hpc_gemm_bf16xfp32_select_splitk(m, n, k, int(bool(use_splitk)))
    # The k-splits reduce through cluster shared memory: no `split_y` scratch (reference
    # entry.cc:116-129) is allocated and `split_flag` is validated but never written.
    if split_flag is not None:
        _require(split_flag.dtype == torch.int32 and split_flag.is_cuda, "split_flag must be cuda int32")
    y = torch.empty((m, n), dtype=torch.float32 if use_fp32_output else torch.bfloat16,
                    device=x.device)
    _check_rc(_lib.hpc_gemm_bf16xfp32_async(
        _ptr(y), None, _ptr(split_flag), _ptr(x), _ptr(w_high),
        _ptr(w_low), m, n, k, float(scale), int(bool(use_fp32_output)), split_k, 128, 1,
        split_flag.stride(0) if split_flag is not None else 0,
        _stream_of(x)), "gemm_bf16xfp32")
    return y


_ops.define(
    "gemm_bf16xfp32(Tensor x, Tensor w_high, Tensor w_low, "
    "float scale, bool use_fp32_output, bool use_splitk, Tensor? split_flag) -> (Tensor)")
_ops.impl("gemm_bf16xfp32", _gemm_bf16xfp32_impl, "CUDA")


def get_gemm_bf16xfp32_workspace(max_weight_hidden_size: int, max_tokens: int = 131072) -> Tensor:
    """Zeroed split-k counter workspace (same sizing as reference hpc/gemm.py:7-13)."""
    min_tile_m = 16
    min_tile_n = 64
    nm_max = (max_tokens + min_tile_m - 1) // min_tile_m
    nn_max = (max_weight_hidden_size + min_tile_n - 1) // min_tile_n
    return torch.zeros((nm_max, nn_max), dtype=torch.int32, device="cuda")


def gemm_bf16xfp32(x: Tensor, w_high: Tensor, w_low: Tensor, scale, use_fp32_output: bool = False,
                   use_splitk: bool = True, split_flag: Tensor = None) -> Tensor:
    """fp32-weight GEMM as two bf16 GEMMs: Y = X @ w_high^T + scale * (X @ w_low^T) with
    w_high = w.bf16, w_low = ((w - w_high) / scale).bf16, scale = 1/256 (reference hpc/gemm.py:16-61).
      x [m, k] bf16; w_high, w_low [n, k] bf16 (n % 64 == 0); returns [m, n] bf16 or fp32.
    `split_flag` (optional, from get_gemm_bf16xfp32_workspace) must be zero and is left zero."""
    return torch.ops.hpc.gemm_bf16xfp32(x, w_high, w_low, float(scale), use_fp32_output, use_splitk,
                                        split_flag)


@torch.library.register_fake("hpc::gemm_bf16xfp32")
def _gemm_bf16xfp32_fake(a, b_high, b_low, scale, use_fp32_output=False, use_splitk=True,
                         split_flag=None):
    dt = torch.float32 if use_fp32_output else a.dtype
    return torch.empty((a.shape[0], b_high.shape[0]), dtype=dt, device=a.device)


def _gemm_blockwise_fp8_impl(x, x_scale, weight, weight_scale, output):
    what = "gemm_blockwise_fp8"
    _require(x.dim() == 2 and weight.dim() == 2, f"{what}: x and weight must be 2-D")
    m, k = x.shape
    n = weight.size(0)
    _require(k % 128 == 0 and 128 <= k <= 65536,
             f"{what}: K ({k}) must be a multiple of 128 in [128, 65536]")
    _require(n > 0 and n % 8 == 0, f"{what}: N ({n}) must be a positive multiple of 8")
    dev = x.device
    _require(x.is_cuda, f"{what}: x must be a cuda tensor")
    for name, t, shape, dtype in (("x", x, (m, k), torch.float8_e4m3fn),
                                  ("x_scale", x_scale, (m, k // 128), torch.float32),
                                  ("weight", weight, (n, k), torch.float8_e4m3fn),
                                  ("weight_scale", weight_scale, ((n + 127) // 128, k // 128),
                                   torch.float32)):
        _require(t.dtype == dtype and tuple(t.shape) == shape and t.device == dev and t.is_contiguous(),
                 f"{what}: {name} must be a contiguous {dtype} tensor of shape {list(shape)} on "
                 f"{dev}, got {t.dtype} {list(t.shape)} on {t.device}")
    if output is None:
        output = torch.empty((m, n), dtype=torch.bfloat16, device=dev)
    _require(output.dtype == torch.bfloat16 and tuple(output.shape) == (m, n) and output.device == dev
             and output.is_contiguous(),
             f"{what}: output must be a contiguous bfloat16 tensor of shape {[m, n]} on {dev}")
    _check_rc(_lib.hpc_gemm_blockwise_fp8_async(_ptr(output), _ptr(x), _ptr(x_scale), _ptr(weight),
                                                _ptr(weight_scale), m, n, k, _stream_of(x)), what)
    return output


_ops.define("gemm_blockwise_fp8(Tensor x, Tensor x_scale, Tensor weight, Tensor weight_scale, "
            "Tensor? output) -> (Tensor)")
_ops.impl("gemm_blockwise_fp8", _gemm_blockwise_fp8_impl, "CUDA")


def gemm_blockwise_fp8(x: Tensor, x_scale: Tensor, weight: Tensor, weight_scale: Tensor,
                       output: Optional[Tensor] = None) -> Tensor:
    """Dense block-scaled FP8 linear layer: y = x . weight^T in bf16 [M, N].
      x e4m3 [M, K] and x_scale f32 [M, K / 128] (as blockwise_fp8_quant returns them);
      weight e4m3 [N, K] (nn.Linear layout) and weight_scale f32 [ceil(N / 128), K / 128] (the
      checkpoint's weight_scale_inv as stored, no padding); all contiguous, 16-byte aligned.
    K % 128 == 0 with 128 <= K <= 65536, N % 8 == 0, any M >= 0.
    Arithmetic, per 128-column K block kb in ascending order: P = the e4m3 tensor-core products
    accumulated over the block's four k = 32 steps from zero; acc = fmaf(P, fl32(x_scale[m, kb] *
    weight_scale[n // 128, kb]), acc). When the problem is split over K (small M; see
    hpc._ffi.lib.hpc_gemm_blockwise_fp8_config) each split does this over its contiguous share of
    the K blocks and the partials are added in fp32 in split order. y = bf16_rn(acc).
    Deterministic: two calls give identical bits. A caller-given `output` is overwritten entirely.
    No allocation beyond the output and no host synchronisation: capturable."""
    return torch.ops.hpc.gemm_blockwise_fp8(x, x_scale, weight, weight_scale, output)


@torch.library.register_fake("hpc::gemm_blockwise_fp8")
def _gemm_blockwise_fp8_fake(x, x_scale, weight, weight_scale, output=None):
    return torch.empty((x.shape[0], weight.shape[0]), dtype=torch.bfloat16, device=x.device)
