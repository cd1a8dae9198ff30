"""Fused RMSNorm -> FP8 quantisation (API of reference hpc/normalization.py): the prologue that
produces the e4m3 activations consumed by the per-tensor FP8 GEMMs and the per-tensor FusedMoE."""
from typing import Tuple, Union

import torch
from torch import Tensor

from . import _ops
from ._ffi import (check as _check_rc, lib as _lib, ptr as _ptr, require as _require,
                   stream_of as _stream_of)


def _fused_rmsnorm_with_scale_impl(input, weight, scale, eps, is_moe):
    # reference src/normalization/entry.cc:20-54, plus the argument checks it leaves out
    _require(input.dtype == torch.bfloat16, "fused_rmsnorm_with_scale: input must be bfloat16")
    _require(input.is_contiguous(), "fused_rmsnorm_with_scale: input must be contiguous")
    _require(input.dim() >= 1, "fused_rmsnorm_with_scale: input must have a hidden dimension")
    hidden = input.shape[-1]
    _require(weight.dtype == torch.bfloat16 and weight.is_contiguous() and weight.numel() == hidden,
             f"fused_rmsnorm_with_scale: weight must be a contiguous bfloat16 tensor of {hidden} "
             f"elements, got {tuple(weight.shape)} {weight.dtype}")
    need = 2 if is_moe else 1
    _require(scale.dtype == torch.float32 and scale.numel() >= need,
             f"fused_rmsnorm_with_scale: scale must be float32 with at least {need} value(s)")
    _require(input.is_cuda and weight.device == input.device and scale.device == input.device,
             "fused_rmsnorm_with_scale: input, weight and scale must be on the same CUDA device")
    batch = input.numel() // hidden if hidden else 0
    output = torch.empty_like(input, dtype=torch.float8_e4m3fn)
    output_fp32 = torch.empty_like(input, dtype=torch.float32)
    output_scale2 = torch.empty_like(input, dtype=torch.float8_e4m3fn)
    _check_rc(_lib.hpc_fused_rmsnorm_with_scale_async(
        _ptr(input), _ptr(weight), _ptr(output), _ptr(output_fp32) if is_moe else None,
        _ptr(output_scale2) if is_moe else None, _ptr(scale), float(eps), batch, hidden,
        int(bool(is_moe)), _stream_of(input)), "fused_rmsnorm_with_scale")
    return output, output_fp32, output_scale2


_ops.define("fused_rmsnorm_with_scale(Tensor input, Tensor weight, Tensor scale, float eps, "
            "bool is_moe) -> (Tensor, Tensor, Tensor)")
_ops.impl("fused_rmsnorm_with_scale", _fused_rmsnorm_with_scale_impl, "CUDA")


def fused_rmsnorm_with_scale(
    a: Tensor,
    weight: Tensor,
    eps: float = torch.finfo(torch.float32).eps,
    scale: Tensor = torch.tensor([1.0], dtype=torch.float32),
    is_moe: bool = False,
) -> Union[Tensor, Tuple[Tensor, Tensor, Tensor]]:
    """RMSNorm of `a` (bf16 [..., H], any H % 8 == 0 up to 16384) times `weight` (bf16, H values in
    any shape), quantised to fp8_e4m3 after dividing by `scale[0]`:
    y = (a * weight) * rsqrt(mean(a^2) + eps) in fp32, out = e4m3(y * (1 / scale[0])), saturated
    at +-448.

    Returns the e4m3 tensor, or with `is_moe` the tuple (y fp32, e4m3 of y / scale[0], e4m3 of
    y / scale[1]); the first e4m3 tensor is the same byte for byte with and without `is_moe`
    (reference hpc/normalization.py:6-41).

    A `scale` on the CPU (the default) is copied to `a`'s device first, as the reference does.
    That copy is the one step that cannot be captured in a CUDA graph: pass a device `scale` to
    capture the call."""
    if scale.device != a.device:
        scale = scale.to(a.device)
    out_fp8, out_fp32, out_fp8_scale2 = torch.ops.hpc.fused_rmsnorm_with_scale(
        a, weight, scale, eps, is_moe)
    return (out_fp32, out_fp8, out_fp8_scale2) if is_moe else out_fp8


@torch.library.register_fake("hpc::fused_rmsnorm_with_scale")
def _fused_rmsnorm_with_scale_fake(input, weight, scale, eps, is_moe):
    # the three tensors the schema declares, whatever is_moe is
    return (torch.empty_like(input, dtype=torch.float8_e4m3fn),
            torch.empty_like(input, dtype=torch.float32),
            torch.empty_like(input, dtype=torch.float8_e4m3fn))
