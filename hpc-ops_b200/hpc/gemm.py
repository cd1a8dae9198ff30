"""BF16 x FP32 route GEMM (API of reference hpc/gemm.py)."""
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
