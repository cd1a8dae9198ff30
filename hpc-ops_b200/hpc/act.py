"""Stand-alone activation / FP8 quantisation operators (API of reference hpc/act.py), including the
masked variants over the per-expert padded (DeepEP low-latency) layout [E * T_max, 2C], which read
and write only each expert's first num_per_expert[e] rows."""
from typing import Optional, Tuple

import torch
from torch import Tensor

from . import _ops
from ._ffi import (check as _check_rc, lib as _lib, ptr as _ptr, require as _require,
                   stream_of as _stream_of)


def _act_mul_and_quant_impl(input, scale, use_bf16_mul, output):
    # reference src/activation/entry.cc:17-50
    _require(input.is_cuda and scale.is_cuda, "input and scale must be cuda tensors")
    _require(input.dtype == torch.bfloat16, "input dtype must be bfloat16")
    _require(input.is_contiguous(), "input tensor must be contiguous")
    _require(scale.dtype == torch.float32 and scale.numel() >= 1, "scale must be a float32 tensor")
    num_col = input.shape[-1]
    num_row = input.numel() // num_col if num_col else 0
    shape = list(input.shape)
    shape[-1] //= 2
    if output is None:
        output = torch.empty(shape, dtype=torch.float8_e4m3fn, device=input.device)
    else:
        _require(output.is_cuda and output.is_contiguous() and output.dtype == torch.float8_e4m3fn
                 and output.numel() == num_row * (num_col // 2),
                 "output must be a contiguous cuda fp8_e4m3 tensor of shape [..., C]")
    _check_rc(_lib.hpc_act_mul_and_quant_async(_ptr(output), _ptr(input), _ptr(scale), num_row,
                                               num_col, int(bool(use_bf16_mul)), _stream_of(input)),
              "act_mul_and_quant")
    return output


_DTYPE_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def _scaled_fp8_quant_impl(input, scale, output):
    # reference src/activation/entry.cc:158-202
    _require(input.is_cuda, "input must be a CUDA tensor")
    _require(input.is_contiguous(), "input must be contiguous")
    _require(input.numel() > 0, "input must be non-empty")
    _require(input.dtype in _DTYPE_CODE, "input dtype must be float32, float16, or bfloat16")
    if output is None:
        output = torch.empty_like(input, dtype=torch.float8_e4m3fn)
    _require(output.is_cuda, "output must be a CUDA tensor")
    _require(output.is_contiguous(), "output must be contiguous")
    _require(output.shape == input.shape, "output shape must match input shape")
    _require(output.dtype == torch.float8_e4m3fn, "output dtype must be float8_e4m3fn")
    _require(scale is not None, "scale is required for scaled_fp8_quant")
    _require(scale.is_cuda, "scale must be a CUDA tensor")
    _require(scale.dtype == torch.float32, "scale dtype must be float32")
    _require(scale.numel() == 1, "scale must contain one element")
    _check_rc(_lib.hpc_scaled_fp8_quant_async(_ptr(output), _ptr(input), _ptr(scale), input.numel(),
                                              _DTYPE_CODE[input.dtype], _stream_of(input)),
              "scaled_fp8_quant")
    return output, scale


def _masked_args(what, input, num_per_expert, col_multiple):
    # reference src/activation/entry.cc:52-156, plus the layout checks it leaves out
    _require(input.is_cuda and num_per_expert.is_cuda and num_per_expert.device == input.device,
             f"{what}: input and num_per_expert must be on the same CUDA device")
    _require(input.dtype == torch.bfloat16 and input.dim() == 2 and input.is_contiguous(),
             f"{what}: input must be a contiguous bfloat16 [N, 2C] tensor")
    _require(num_per_expert.dtype == torch.int32 and num_per_expert.dim() == 1
             and num_per_expert.is_contiguous() and num_per_expert.numel() >= 1,
             f"{what}: num_per_expert must be a contiguous int32 [E] tensor")
    n, two_c = input.shape
    c = two_c // 2
    _require(two_c % 2 == 0 and c > 0 and c % col_multiple == 0,
             f"{what}: intermediate size {c} must be a positive multiple of {col_multiple}")
    e = num_per_expert.numel()
    _require(n % e == 0, f"{what}: rows ({n}) must be a multiple of the number of experts ({e})")
    return n, c, n // e


def _check_out(what, name, t, shape, dtype, device):
    _require(t.dtype == dtype and tuple(t.shape) == tuple(shape) and t.device == device
             and t.is_contiguous(),
             f"{what}: {name} must be a contiguous {dtype} tensor of shape {list(shape)} on "
             f"{device}, got {t.dtype} {list(t.shape)} on {t.device}")


def _masked_act_mul_and_quant_impl(input, scale, num_per_expert, output):
    what = "masked_act_mul_and_quant"
    n, c, t_max = _masked_args(what, input, num_per_expert, 8)
    _require(scale.is_cuda and scale.device == input.device and scale.dtype == torch.float32
             and scale.numel() == 1, f"{what}: scale must be one float32 value on the input's device")
    if output is None:
        output = torch.empty((n, c), dtype=torch.float8_e4m3fn, device=input.device)
    _check_out(what, "output", output, (n, c), torch.float8_e4m3fn, input.device)
    _check_rc(_lib.hpc_masked_act_mul_and_quant_async(
        _ptr(output), _ptr(input), _ptr(scale), _ptr(num_per_expert), n, c, t_max,
        _stream_of(input)), what)
    return output


def _masked_act_mul_and_blockwise_quant_impl(input, num_per_expert, output, output_scale):
    what = "masked_act_mul_and_blockwise_quant"
    n, c, t_max = _masked_args(what, input, num_per_expert, 128)
    if output is None:
        output = torch.empty((n, c), dtype=torch.float8_e4m3fn, device=input.device)
    if output_scale is None:
        output_scale = torch.empty((n, c // 128), dtype=torch.float32, device=input.device)
    _check_out(what, "output", output, (n, c), torch.float8_e4m3fn, input.device)
    _check_out(what, "output_scale", output_scale, (n, c // 128), torch.float32, input.device)
    _check_rc(_lib.hpc_masked_act_mul_and_blockwise_quant_async(
        _ptr(output), _ptr(output_scale), _ptr(input), _ptr(num_per_expert), n, c, t_max,
        _stream_of(input)), what)
    return output, output_scale


def _blockwise_fp8_quant_impl(input, output, output_scale):
    what = "blockwise_fp8_quant"
    _require(input.is_cuda and input.dtype == torch.bfloat16 and input.dim() == 2,
             f"{what}: input must be a bfloat16 [M, K] cuda tensor")
    m, k = input.shape
    _require(k % 128 == 0 and k > 0, f"{what}: K ({k}) must be a positive multiple of 128")
    _require(input.stride(1) == 1 and (m <= 1 or input.stride(0) % 8 == 0),
             f"{what}: input rows must be contiguous with a row stride that is a multiple of 8")
    if output is None:
        output = torch.empty((m, k), dtype=torch.float8_e4m3fn, device=input.device)
    if output_scale is None:
        output_scale = torch.empty((m, k // 128), dtype=torch.float32, device=input.device)
    _check_out(what, "output", output, (m, k), torch.float8_e4m3fn, input.device)
    _check_out(what, "output_scale", output_scale, (m, k // 128), torch.float32, input.device)
    ld = input.stride(0) if m > 1 else k
    _check_rc(_lib.hpc_blockwise_fp8_quant_async(_ptr(output), _ptr(output_scale), _ptr(input), m,
                                                  k, ld, _stream_of(input)), what)
    return output, output_scale


_ops.define("act_mul_and_quant(Tensor input, Tensor scale, bool use_bf16_mul, Tensor? output) -> "
            "(Tensor)")
_ops.impl("act_mul_and_quant", _act_mul_and_quant_impl, "CUDA")
_ops.define("scaled_fp8_quant(Tensor input, Tensor? scale, Tensor? output) -> (Tensor, Tensor)")
_ops.impl("scaled_fp8_quant", _scaled_fp8_quant_impl, "CUDA")
_ops.define("masked_act_mul_and_quant(Tensor input, Tensor scale, Tensor num_per_expert, "
            "Tensor? output) -> (Tensor)")
_ops.impl("masked_act_mul_and_quant", _masked_act_mul_and_quant_impl, "CUDA")
_ops.define("masked_act_mul_and_blockwise_quant(Tensor input, Tensor num_per_expert, Tensor? output, "
            "Tensor? output_scale) -> (Tensor output, Tensor output_scale)")
_ops.impl("masked_act_mul_and_blockwise_quant", _masked_act_mul_and_blockwise_quant_impl, "CUDA")
_ops.define("blockwise_fp8_quant(Tensor input, Tensor? output, Tensor? output_scale) -> "
            "(Tensor output, Tensor output_scale)")
_ops.impl("blockwise_fp8_quant", _blockwise_fp8_quant_impl, "CUDA")


def act_mul_and_quant(gate_up: Tensor, scale: Tensor, use_bf16_mul: bool = True,
                      output: Tensor = None) -> Tensor:
    """silu(gate_up[:, :C]) * gate_up[:, C:] * scale[0] -> fp8_e4m3 [N, C]; gate_up bf16 [N, 2C]
    (reference hpc/act.py:7-35). With `use_bf16_mul` the product is formed in bf16 as the
    reference kernel does."""
    return torch.ops.hpc.act_mul_and_quant(gate_up, scale, use_bf16_mul, output)


def scaled_fp8_quant(input: Tensor, scale: Optional[Tensor] = None,
                     output: Optional[Tensor] = None) -> Tuple[Tensor, Tensor]:
    """Static per-tensor FP8 quantisation: (input / scale[0]).to(fp8_e4m3); returns (output, scale)
    (reference hpc/act.py scaled_fp8_quant; scale is required, src/activation/entry.cc:179)."""
    return torch.ops.hpc.scaled_fp8_quant(input, scale, output)


def masked_act_mul_and_quant(gate_up: Tensor, scale: Tensor, num_per_expert: Tensor,
                             output: Optional[Tensor] = None) -> Tensor:
    """silu(gate) * up * scale[0] -> fp8_e4m3 [N, C] over the per-expert padded layout
    gate_up bf16 [N = E * T_max, 2C] (C % 8 == 0), computed in fp32 as act_mul_and_quant with
    use_bf16_mul=False. Row e * T_max + t is valid when t < clamp(num_per_expert[e], 0, T_max)
    (num_per_expert int32 [E] on the device); only valid rows are read and written, so the other
    rows of a provided `output` keep their contents (reference hpc/act.py:37-67)."""
    return torch.ops.hpc.masked_act_mul_and_quant(gate_up, scale, num_per_expert, output)


def masked_act_mul_and_blockwise_quant(gate_up: Tensor, num_per_expert: Tensor,
                                       output: Optional[Tensor] = None,
                                       output_scale: Optional[Tensor] = None
                                       ) -> Tuple[Tensor, Tensor]:
    """The masked layout of masked_act_mul_and_quant with 1x128 blockwise quantisation
    (C % 128 == 0): per (row, 128 columns) of v = silu(gate) * up, sc = amax|v| / 448 and
    out = e4m3(v / (sc + 1e-8)); returns (out [N, C], sc f32 row-major [N, C / 128]). Invalid rows
    of provided outputs keep their contents (reference hpc/act.py:70-105)."""
    return torch.ops.hpc.masked_act_mul_and_blockwise_quant(gate_up, num_per_expert, output,
                                                            output_scale)


def blockwise_fp8_quant(input: Tensor, output: Optional[Tensor] = None,
                        output_scale: Optional[Tensor] = None) -> Tuple[Tensor, Tensor]:
    """1x128 blockwise FP8 quantisation of bf16 activations `input` [M, K] (K % 128 == 0, rows
    contiguous, row stride a multiple of 8 elements). Per (row, 128 columns), in fp32:
    sc = amax|v| / 448, out = e4m3_rn_satfinite(v * (1 / (sc + 1e-8))) -- the arithmetic of
    masked_act_mul_and_blockwise_quant without the SiLU * mul. Returns (out e4m3 [M, K],
    sc f32 [M, K / 128]), both contiguous: the (x, x_scale) pair gemm_blockwise_fp8 and
    fuse_moe_blockwise_fp8 take. Caller-given outputs must have exactly these dtypes, shapes and the
    input's device, and be contiguous. No allocation beyond the outputs and no host
    synchronisation: capturable."""
    return torch.ops.hpc.blockwise_fp8_quant(input, output, output_scale)


@torch.library.register_fake("hpc::act_mul_and_quant")
def _act_mul_and_quant_fake(input, scale, use_bf16_mul, output):
    shape = list(input.shape)
    shape[-1] //= 2
    return torch.empty(shape, dtype=torch.float8_e4m3fn, device=input.device)


@torch.library.register_fake("hpc::scaled_fp8_quant")
def _scaled_fp8_quant_fake(input, scale, output):
    return torch.empty_like(input, dtype=torch.float8_e4m3fn), scale


@torch.library.register_fake("hpc::masked_act_mul_and_quant")
def _masked_act_mul_and_quant_fake(input, scale, num_per_expert, output):
    return torch.empty(input.shape[0], input.shape[1] // 2, dtype=torch.float8_e4m3fn,
                       device=input.device)


@torch.library.register_fake("hpc::masked_act_mul_and_blockwise_quant")
def _masked_act_mul_and_blockwise_quant_fake(input, num_per_expert, output, output_scale):
    n, c = input.shape[0], input.shape[1] // 2
    return (torch.empty(n, c, dtype=torch.float8_e4m3fn, device=input.device),
            torch.empty(n, c // 128, dtype=torch.float32, device=input.device))


@torch.library.register_fake("hpc::blockwise_fp8_quant")
def _blockwise_fp8_quant_fake(input, output, output_scale):
    m, k = input.shape
    return (torch.empty(m, k, dtype=torch.float8_e4m3fn, device=input.device),
            torch.empty(m, k // 128, dtype=torch.float32, device=input.device))
