"""Fused AllReduce + residual + RMSNorm (API of reference hpc/allreduce.py)."""
from typing import Any as _Any, Optional as _Optional, Sequence as _Sequence, Tuple as _Tuple

import torch

from . import _ops
from ._ffi import (check as _check_rc, lib as _lib, ptr as _ptr, require as _require,
                   stream_of as _stream_of)
from .communicator import MulticastCommunicator
from .multicast_handle import MulticastHandle, _find_handle

import ctypes as _ctypes
import os as _os

# world sizes up to which the high-throughput path prefers direct P2P loads/stores over NVLS
_P2P_MAX_WORLD = int(_os.environ.get("HPC_B200_AR_P2P_MAX_WORLD", "2"))


def _ht_impl(input, mc_input, in_residual, weight, signal, rank, world_size, num_max_blocks,
             rms_norm_eps, output, mc_output, out_residual):
    # validation follows reference src/allreduce/entry.cc:14-76 (hidden size is not restricted to
    # {4096, 5120, 7168} in this build)
    for t, name in ((input, "input"), (mc_input, "mc_input"), (in_residual, "input residual"),
                    (output, "output"), (mc_output, "mc_output"), (out_residual, "output residual"),
                    (weight, "weight"), (signal, "signal")):
        _require(t.is_contiguous(), f"{name} tensor must be contigous")
    for t, name in ((input, "input"), (in_residual, "residual"), (output, "output"),
                    (out_residual, "output residual"), (weight, "weight")):
        _require(t.dtype == torch.bfloat16, f"{name} tensor data type must be bfloat16")
    _require(signal.dtype == torch.int64, "signal tensor data type must be int64")
    hidden = input.size(-1)
    num_tokens = input.numel() // hidden
    for t in (input, mc_input, in_residual, output, mc_output, out_residual, weight):
        _require(t.data_ptr() % 16 == 0, "pointer must be aligned to 16")
    mc_in = mc_input.data_ptr()
    mc_out = mc_output.data_ptr()
    peers_in = peers_out = None
    no_mc = world_size > 1 and (mc_in == input.data_ptr() or mc_out == output.data_ptr())
    hi = ho = None
    if world_size > 1 and (no_mc or world_size <= _P2P_MAX_WORLD):
        hi, ho = _find_handle(input.data_ptr()), _find_handle(output.data_ptr())
    if no_mc or (hi is not None and ho is not None):
        # P2P variant over the peers' symmetric buffers: the only choice without an NVLS mapping,
        # and the cheaper one on two GPUs (each link direction carries N/2 bytes; the in-switch
        # reduction pulls every rank's full input, 1.5 N per direction at W=2 -- DESIGN.md 3.7)
        _require(hi is not None and ho is not None,
                 "allreduce without multicast needs buffers from hpc.empty_multimem")
        off_i = input.data_ptr() - hi.data_buffer_list_[hi.rank].data_ptr()
        off_o = output.data_ptr() - ho.data_buffer_list_[ho.rank].data_ptr()
        peers_in = (_ctypes.c_int64 * world_size)(*[int(p) + off_i for p in hi.data_buffer_ptrs_])
        peers_out = (_ctypes.c_int64 * world_size)(*[int(p) + off_o for p in ho.data_buffer_ptrs_])
        mc_in = mc_out = None
    _check_rc(_lib.hpc_fuse_allreduce_rmsnorm_high_throughput_p2p_async(
        _ptr(input), mc_in, _ptr(in_residual), _ptr(weight), _ptr(output), mc_out,
        _ptr(out_residual), _ptr(signal), peers_in, peers_out, int(rank), int(world_size),
        int(num_max_blocks), float(rms_norm_eps), num_tokens, hidden, _stream_of(input)),
        "fuse_allreduce_rmsnorm_high_throughput")


def _ll_impl(input_x, multicast_x, data_buffer_ptrs, multinode_x, buffer_flags, world_size, rank,
             rmsnorm_fusion, launch_with_pdl, use_two_shot, output_x, residual_out, residual_in,
             weight_gamma, rms_norm_eps):
    # reference src/allreduce/entry.cc:78-197
    for t, name in ((input_x, "input"), (multinode_x, "workspace"), (output_x, "output"),
                    (residual_out, "residual_out"), (residual_in, "residual_in"),
                    (weight_gamma, "weight")):
        _require(t.is_cuda and t.is_contiguous(), f"{name} must be a contiguous cuda tensor")
    _require(input_x.dtype == torch.bfloat16, "input tensor data type must be bfloat16")
    _require(buffer_flags.dtype in (torch.uint32, torch.int32) and buffer_flags.numel() >= 9,
             "buffer_flags must be uint32[9]")
    hidden = input_x.size(-1)
    num_tokens = input_x.numel() // hidden
    mc = multicast_x.data_ptr() if multicast_x is not None else 0
    if mc == multinode_x.data_ptr():
        mc = 0  # no NVLS mapping: broadcast with P2P stores
    # use_two_shot=True is the reference protocol; False lets the kernel take the one-shot protocol
    # when the batch is small and the workspace is large enough (it decides from buffer_flags[2])
    _check_rc(_lib.hpc_fuse_allreduce_rmsnorm_low_latency_ex_async(
        int(world_size), int(rank), num_tokens, hidden, _ptr(data_buffer_ptrs), _ptr(multinode_x),
        mc or None, _ptr(buffer_flags), int(bool(rmsnorm_fusion)), int(bool(launch_with_pdl)),
        _ptr(input_x), _ptr(residual_in), _ptr(weight_gamma), float(rms_norm_eps),
        _ptr(residual_out), _ptr(output_x), 0, 1 if use_two_shot else 0, _stream_of(input_x)),
        "fuse_allreduce_rmsnorm_low_latency")


_ops.define(
    "fuse_allreduce_rmsnorm_high_throughput(Tensor input, Tensor mc_input, Tensor in_residual, "
    "Tensor weight, Tensor signal, int rank, int world_size, int num_max_blocks, float "
    "rms_norm_eps, Tensor! output, Tensor! mc_output, Tensor! out_residual) -> ()")
_ops.impl("fuse_allreduce_rmsnorm_high_throughput", _ht_impl, "CUDA")
_ops.define(
    "fuse_allreduce_rmsnorm_low_latency(Tensor input_x, Tensor multicast_x, "
    "Tensor data_buffer_ptrs, Tensor! multinode_x, Tensor buffer_flags, "
    "int world_size, int rank, bool rmsnorm_fusion, bool launch_with_pdl, bool use_two_shot, "
    "Tensor! output_x, Tensor! residual_out, Tensor residual_in, "
    "Tensor weight_gamma, float rms_norm_eps) -> ()")
_ops.impl("fuse_allreduce_rmsnorm_low_latency", _ll_impl, "CUDA")


def fuse_allreduce_rmsnorm_high_throughput(
    x: torch.Tensor, multicast_x: torch.Tensor, residual: torch.Tensor, weight: torch.Tensor,
    rms_norm_eps: float, signal: torch.Tensor, rank: int, world_size: int, num_max_blocks: int,
    output_x: _Optional[torch.Tensor] = None, output_multicast_x: _Optional[torch.Tensor] = None,
    output_residual: _Optional[torch.Tensor] = None,
) -> None:
    """RMSNorm(AllReduce(x) + residual, weight) over this rank's token slice; the normalised rows
    are broadcast into every rank's symmetric output buffer (reference hpc/allreduce.py:7-75).
      x / output_x: this rank's slice [n, hidden] of symmetric buffers from `empty_multimem`;
      multicast_x / output_multicast_x: the same slices at the multicast address;
      signal: `MulticastHandle.signal_buffer_ptrs_dev`. All ranks must pass the same num_max_blocks."""
    if output_x is None:
        output_x = x
    if output_multicast_x is None:
        output_multicast_x = multicast_x
    if output_residual is None:
        output_residual = residual
    torch.ops.hpc.fuse_allreduce_rmsnorm_high_throughput(
        x, multicast_x, residual, weight, signal, rank, world_size, num_max_blocks, rms_norm_eps,
        output_x, output_multicast_x, output_residual)


def fuse_allreduce_rmsnorm_low_latency(
    input_x: torch.Tensor, multicast_x: torch.Tensor, data_buffer_ptrs: torch.Tensor,
    multinode_x: torch.Tensor, buffer_flags: torch.Tensor, world_size: int, rank: int,
    residual_in: torch.Tensor, weight_gamma: torch.Tensor, rms_norm_eps: float, num_max_blocks: int,
    output_x: _Optional[torch.Tensor] = None, residual_out: _Optional[torch.Tensor] = None,
    launch_with_pdl: bool = True, use_two_shot: bool = False,
) -> None:
    """Low-latency (Lamport) fused AllReduce + residual + RMSNorm: every rank ends with the full
    [tokens, hidden] output (reference hpc/allreduce.py:78-123). `multinode_x` is the
    triple-buffered workspace initialised to 0x80000000 words, `buffer_flags` its uint32[9] state.
    use_two_shot=True forces the reference's two-shot protocol; by default small batches whose
    [tokens][world][hidden] image fits one workspace buffer take the one-shot protocol."""
    if output_x is None:
        output_x = input_x
    if residual_out is None:
        residual_out = residual_in
    torch.ops.hpc.fuse_allreduce_rmsnorm_low_latency(
        input_x, multicast_x, data_buffer_ptrs, multinode_x, buffer_flags, world_size, rank, True,
        launch_with_pdl, bool(use_two_shot), output_x, residual_out, residual_in, weight_gamma,
        rms_norm_eps)


def empty_multimem(multicomm, *size: _Any, dtype: _Optional[torch.dtype] = None,
                   device: _Optional[torch.device] = None) -> _Tuple[torch.Tensor, MulticastHandle]:
    """Allocate a symmetric (and, where supported, multicast) buffer over single-node NVLink.
    Returns this rank's tensor and its MulticastHandle (reference hpc/allreduce.py:164-200)."""
    if len(size) == 1 and isinstance(size[0], _Sequence):
        size = tuple(size[0])
    else:
        size = tuple(size)
    if dtype is None:
        dtype = torch.get_default_dtype()
    hdl = MulticastHandle(multicomm, size, dtype)
    return hdl.get_buffer(hdl.rank, size, dtype=dtype), hdl
