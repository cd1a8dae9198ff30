"""Fused token sampler (API of reference hpc/sampler.py): repetition penalty, temperature, optional
softmax, top-k, top-p and Gumbel-max sampling of one token per row in one sm_90a kernel, and the
penalty-mask write-back. Fused speculative sampling (no reference counterpart): acceptance of
multi-token-prediction drafts and the recovered or bonus token. No host synchronisation; capturable
in a CUDA graph."""
import ctypes
from enum import IntEnum
from typing import Optional, Tuple, Union

import torch
from torch import Tensor

from . import _ops
from ._ffi import (check as _check_rc, lib as _lib, ptr as _ptr, require as _require,
                   stream_of as _stream_of)


class SoftmaxPolicy(IntEnum):
    """Where the sampler computes probabilities.

    * ``NONE``: none; Gumbel-max runs on the (penalised, tempered) logits x.
    * ``BEFORE_TOPK``: p = softmax(x) over the whole vocabulary; top-p cuts on it.
    * ``AFTER_TOPK``: p = softmax over the top-K candidates only; top-p cuts on it.

    Candidates are always the top-K of x (exp is monotonic, so this is the top-K of p too).
    """

    NONE = 0
    BEFORE_TOPK = 1
    AFTER_TOPK = 2


_MAX_VOCAB = 262144


def _per_row_arg(value, name: str):
    """A sampler parameter as the op takes it: a [B] tensor with a zero scalar beside it, or no
    tensor and the Python scalar itself."""
    if not isinstance(value, Tensor):
        return None, value
    if value.dtype == torch.float32:
        return value, 0.0
    if value.dtype in (torch.int32, torch.int64):
        return value, 0
    raise ValueError(f"fused_sampler: {name} given as a {value.dtype} tensor; use float32 "
                     "(int32 or int64 for topk)")


def _check_logits(logits: Tensor, max_topk: int) -> Tuple[int, int, int]:
    _require(logits.is_cuda and logits.dim() == 2, "logits must be a 2-D CUDA tensor")
    _require(logits.dtype in (torch.float32, torch.bfloat16), "logits dtype must be float32 or bfloat16")
    _require(logits.stride(1) == 1, "logits must have stride(1) == 1")
    B, V = logits.shape
    _require(V % 8 == 0 and max_topk <= V <= _MAX_VOCAB,
             f"vocab size {V} must be a multiple of 8 in [{max_topk}, {_MAX_VOCAB}]")
    esz = logits.element_size()
    _require(logits.data_ptr() % 16 == 0 and (logits.stride(0) * esz) % 16 == 0 and logits.stride(0) >= V,
             "logits rows must be 16-byte aligned")
    return B, V, 0 if logits.dtype == torch.float32 else 1


def _check_row_param(t: Optional[Tensor], name: str, B: int, dtypes, device):
    if t is None:
        return
    _require(t.device == device, f"{name} must be on the device of logits")
    _require(t.dtype in dtypes, f"{name} dtype must be one of {dtypes}")
    _require(t.dim() == 1 and t.shape[0] == B and t.is_contiguous(),
             f"{name} must be a contiguous [batch_size={B}] tensor")


def _check_noise(gumbel_noise: Optional[Tensor], B: int, V: int, seed: int, device):
    if gumbel_noise is None:
        _require(seed > 0, f"sampling with the kernel's own noise needs a seed >= 1 (seed={seed}); "
                 "pass gumbel_noise to sample without one")
        return
    _require(gumbel_noise.device == device and gumbel_noise.dtype == torch.float32
             and gumbel_noise.is_contiguous() and tuple(gumbel_noise.shape) == (B, V),
             f"gumbel_noise must be a contiguous float32 [{B}, {V}] tensor on the device of logits")


def _fused_sampler_impl(logits, penalty_mask, slot_id, repetition_penalty, repetition_penalty_val,
                        temperature, temperature_val, softmax_policy, topk, topk_val, topp, topp_val,
                        max_topk, gumbel_noise=None, seed=0):
    _require(max_topk in (32, 64), f"max_topk is {max_topk}; the kernels are built for 32 and 64")
    B, V, dtype = _check_logits(logits, max_topk)
    dev = logits.device
    _require(softmax_policy in (0, 1, 2), f"softmax_policy {softmax_policy} is not a SoftmaxPolicy value")
    _require((penalty_mask is None) == (slot_id is None),
             "penalty_mask and slot_id go together: pass both or neither")
    if penalty_mask is not None:
        _require(penalty_mask.device == dev and penalty_mask.dtype == torch.uint8 and penalty_mask.dim() == 2
                 and penalty_mask.is_contiguous() and penalty_mask.shape[1] >= V // 8
                 and penalty_mask.shape[0] >= B,
                 "penalty_mask must be a contiguous uint8 [MAX_BS >= batch, >= V/8] tensor")
        # the write-back ORs the sampled bit into the aligned 4-byte word holding its byte, so the
        # mask must cover whole words (widen its rows to a multiple of 4 bytes if it does not)
        _require(penalty_mask.data_ptr() % 4 == 0 and penalty_mask.numel() % 4 == 0,
                 f"penalty_mask must start 4-byte aligned and hold a multiple of 4 bytes "
                 f"(it holds {penalty_mask.numel()})")
        _check_row_param(slot_id, "slot_id", B, (torch.int32,), dev)
    _check_row_param(repetition_penalty, "repetition_penalty", B, (torch.float32,), dev)
    _check_row_param(temperature, "temperature", B, (torch.float32,), dev)
    _check_row_param(topk, "topk", B, (torch.int32, torch.int64), dev)
    _check_row_param(topp, "topp", B, (torch.float32,), dev)
    # a feature is on when its tensor is given or its scalar is positive
    penalising = repetition_penalty is not None or repetition_penalty_val > 0
    top_k_on = topk is not None or topk_val > 0
    top_p_on = topp is not None or topp_val > 0
    _require(penalty_mask is not None or not penalising,
             "a repetition penalty needs the penalty_mask (and slot_id) that says which tokens it hits")
    if top_p_on:
        _require(top_k_on, "top-p cuts the top-k candidates: set topk as well")
        _require(softmax_policy != 0, "top-p needs probabilities: choose BEFORE_TOPK or AFTER_TOPK")
    else:
        # without top-p a softmax cannot change which token wins
        _require(softmax_policy == 0, "a softmax policy other than NONE is only meaningful with top-p")
    _check_noise(gumbel_noise, B, V, seed, dev)
    out = torch.empty(B, 1, dtype=torch.int32, device=dev)
    _check_rc(_lib.hpc_fused_sampler_async(
        _ptr(out), _ptr(logits), logits.stride(0), dtype, B, V, _ptr(penalty_mask),
        V // 8 if penalty_mask is None else penalty_mask.stride(0), _ptr(slot_id),
        _ptr(repetition_penalty), float(repetition_penalty_val), _ptr(temperature),
        float(temperature_val), int(softmax_policy), _ptr(topk),
        int(topk is not None and topk.dtype == torch.int64), int(topk_val), _ptr(topp), float(topp_val),
        int(max_topk), _ptr(gumbel_noise), max(int(seed), 0), _stream_of(logits)), "fused_sampler")
    return out


def _fused_sampler_temperature_sample_impl(logits, temperature, temperature_val, gumbel_noise=None,
                                           draft_token_ids=None, seed=0):
    B, V, dtype = _check_logits(logits, 1)
    dev = logits.device
    _check_row_param(temperature, "temperature", B, (torch.float32,), dev)
    if draft_token_ids is not None:
        _require(draft_token_ids.device == dev and draft_token_ids.dtype == torch.int64
                 and draft_token_ids.dim() == 1 and draft_token_ids.shape[0] == B
                 and draft_token_ids.is_contiguous(),
                 f"draft_token_ids must be a contiguous int64 [batch_size={B}] tensor")
    _check_noise(gumbel_noise, B, V, seed, dev)
    out = torch.empty(B, 1, dtype=torch.int32, device=dev)
    _check_rc(_lib.hpc_fused_sampler_temperature_sample_async(
        _ptr(out), _ptr(logits), logits.stride(0), dtype, B, V, _ptr(temperature),
        float(temperature_val), _ptr(gumbel_noise), _ptr(draft_token_ids), max(int(seed), 0),
        _stream_of(logits)), "fused_sampler_temperature_sample")
    return out


_ops.define("fused_sampler(Tensor logits, Tensor? penalty_mask, Tensor? slot_id, "
            "Tensor? repetition_penalty, float repetition_penalty_val, Tensor? temperature, "
            "float temperature_val, int softmax_policy, Tensor? topk, int topk_val, Tensor? topp, "
            "float topp_val, int max_topk, Tensor? gumbel_noise=None, int seed=0) -> Tensor")
_ops.impl("fused_sampler", _fused_sampler_impl, "CUDA")
_ops.define("fused_sampler_temperature_sample(Tensor logits, Tensor? temperature, "
            "float temperature_val, Tensor? gumbel_noise=None, Tensor? draft_token_ids=None, "
            "int seed=0) -> Tensor")
_ops.impl("fused_sampler_temperature_sample", _fused_sampler_temperature_sample_impl, "CUDA")


@torch.library.register_fake("hpc::fused_sampler")
def _fused_sampler_fake(logits, penalty_mask, slot_id, repetition_penalty, repetition_penalty_val,
                        temperature, temperature_val, softmax_policy, topk, topk_val, topp, topp_val,
                        max_topk, gumbel_noise=None, seed=0):
    return logits.new_empty((logits.shape[0], 1), dtype=torch.int32)


@torch.library.register_fake("hpc::fused_sampler_temperature_sample")
def _fused_sampler_temperature_sample_fake(logits, temperature, temperature_val, gumbel_noise=None,
                                           draft_token_ids=None, seed=0):
    return logits.new_empty((logits.shape[0], 1), dtype=torch.int32)


def fused_sampler(
    logits: Tensor,
    *,
    penalty_mask: Optional[Tensor] = None,
    slot_id: Optional[Tensor] = None,
    repetition_penalty: Union[Tensor, float] = 0.0,
    temperature: Union[Tensor, float] = 0.0,
    softmax_policy: SoftmaxPolicy = SoftmaxPolicy.NONE,
    topk: Union[Tensor, int] = 0,
    topp: Union[Tensor, float] = 0.0,
    max_topk: int = 32,
    gumbel_noise: Optional[Tensor] = None,
    draft_token_ids: Optional[Tensor] = None,
    seed: int = 0,
) -> Tensor:
    """Sample one token per row of `logits` [B, V] (float32 or bfloat16) -> int32 [B, 1].

    Per row b, on x = float(logits[b]): the repetition penalty (where bit v of
    penalty_mask[slot_id[b]] is set and rp_b > 0, positive x is divided by rp_b and the rest
    multiplied), then x / t_b where t_b > 0. Then the top-K_b of x (K_b = topk_b if
    1 <= topk_b <= max_topk, else max_topk; ties go to the smaller token id), probabilities by
    `softmax_policy`, top-p (keep rank 0 and every rank whose exclusive cumulative p is below
    topp_b), and the token with the largest value + Gumbel noise (x for NONE, log p otherwise).
    The sampled token's bit is OR-ed into penalty_mask[slot_id[b]].

    Tokens outside the top-max_topk are never drawn. Per-row parameters are scalars or [B]
    tensors (float32; topk int32 or int64). `gumbel_noise` [B, V] float32 makes the result
    deterministic; without it the kernel draws Philox4x32-10 noise keyed by `seed` (> 0) and a
    per-stream launch counter, so successive calls and graph replays draw fresh noise.

    With temperature alone (penalty, top-k, top-p and softmax off, temperature a tensor or a
    positive scalar) the call takes a lighter kernel that adds noise to every token;
    `draft_token_ids` [B] int64 (that token of row b is excluded when in [0, V)) is only accepted
    there, and rows with t_b <= 0 or NaN return the argmax of the logits (draft token excluded).
    The penalty mask must start 4-byte aligned and hold a multiple of 4 bytes.
    """
    policy = SoftmaxPolicy(int(softmax_policy))
    if max_topk not in (32, 64):
        raise ValueError(f"fused_sampler: max_topk is {max_topk}; it must be 32 or 64")

    def off(v):  # a feature given as a Python zero (a tensor always counts as on)
        return not isinstance(v, Tensor) and float(v) == 0.0

    temperature_only = (penalty_mask is None and slot_id is None and policy == SoftmaxPolicy.NONE
                        and off(repetition_penalty) and off(topk) and off(topp)
                        and (isinstance(temperature, Tensor) or float(temperature) > 0.0))
    if temperature_only:
        t, t_val = _per_row_arg(temperature, "temperature")
        return torch.ops.hpc.fused_sampler_temperature_sample(
            logits, t, float(t_val), gumbel_noise, draft_token_ids, seed)
    if draft_token_ids is not None:
        raise ValueError("fused_sampler: draft_token_ids works with temperature alone; this call "
                         "also sets a penalty, top-k, top-p or softmax policy")
    rp, rp_val = _per_row_arg(repetition_penalty, "repetition_penalty")
    t, t_val = _per_row_arg(temperature, "temperature")
    k, k_val = _per_row_arg(topk, "topk")
    p, p_val = _per_row_arg(topp, "topp")
    return torch.ops.hpc.fused_sampler(logits, penalty_mask, slot_id, rp, rp_val, t, t_val, int(policy),
                                       k, k_val, p, p_val, max_topk, gumbel_noise, seed)


_MAX_DRAFT = 8


def _fused_speculative_sampler_impl(target_logits, draft_token_ids, draft_probs, temperature,
                                    temperature_val, uniform=None, gumbel_noise=None, seed=0):
    N, V, dtype = _check_logits(target_logits, 1)
    dev = target_logits.device
    _require(draft_token_ids.device == dev and draft_token_ids.dtype in (torch.int32, torch.int64)
             and draft_token_ids.dim() == 2 and draft_token_ids.is_contiguous(),
             "draft_token_ids must be a contiguous int32 or int64 [batch_size, K] tensor on the "
             "device of target_logits")
    B, K = draft_token_ids.shape
    _require(1 <= K <= _MAX_DRAFT, f"K = {K} draft tokens per request; 1 to {_MAX_DRAFT} are supported")
    _require(N == B * (K + 1), f"target_logits has {N} rows; batch_size {B} x (K + 1) = {B * (K + 1)} "
             "expected (row b * (K + 1) + i is position i of request b)")
    _require(N <= 65535, f"batch_size x (K + 1) = {N} rows exceeds 65535")
    if draft_probs is not None:
        _require(draft_probs.device == dev and draft_probs.dtype == torch.float32
                 and draft_probs.is_contiguous() and tuple(draft_probs.shape) == (B, K, V)
                 and draft_probs.data_ptr() % 16 == 0,
                 f"draft_probs must be a contiguous, 16-byte aligned float32 [{B}, {K}, {V}] tensor "
                 "on the device of target_logits")
    _check_row_param(temperature, "temperature", B, (torch.float32,), dev)
    _require((uniform is None) == (gumbel_noise is None),
             "uniform and gumbel_noise go together: pass both or neither")
    if uniform is None:
        if temperature is not None or temperature_val > 0:
            _require(seed > 0, f"sampling with the kernel's own noise needs a seed >= 1 (seed={seed}); "
                     "pass uniform and gumbel_noise to sample without one")
    else:
        _require(uniform.device == dev and uniform.dtype == torch.float32 and uniform.is_contiguous()
                 and tuple(uniform.shape) == (B, K),
                 f"uniform must be a contiguous float32 [{B}, {K}] tensor on the device of target_logits")
        _require(gumbel_noise.device == dev and gumbel_noise.dtype == torch.float32
                 and gumbel_noise.is_contiguous() and tuple(gumbel_noise.shape) == (N, V)
                 and gumbel_noise.data_ptr() % 16 == 0,
                 f"gumbel_noise must be a contiguous, 16-byte aligned float32 [{N}, {V}] tensor on the "
                 "device of target_logits")
    out = torch.empty(B, K + 1, dtype=torch.int32, device=dev)
    num_accepted = torch.empty(B, dtype=torch.int32, device=dev)
    records = torch.empty(N, 8, dtype=torch.int32, device=dev)  # 32 bytes per row for the kernels
    _check_rc(_lib.hpc_fused_speculative_sampler_async(
        _ptr(out), _ptr(num_accepted), _ptr(records), _ptr(target_logits), target_logits.stride(0), dtype,
        B, K, V, _ptr(draft_token_ids), int(draft_token_ids.dtype == torch.int64), _ptr(draft_probs),
        _ptr(temperature), float(temperature_val), _ptr(uniform), _ptr(gumbel_noise), max(int(seed), 0),
        _stream_of(target_logits)), "fused_speculative_sampler")
    return out, num_accepted


_ops.define("fused_speculative_sampler(Tensor target_logits, Tensor draft_token_ids, Tensor? draft_probs, "
            "Tensor? temperature, float temperature_val, Tensor? uniform=None, Tensor? gumbel_noise=None, "
            "int seed=0) -> (Tensor, Tensor)")
_ops.impl("fused_speculative_sampler", _fused_speculative_sampler_impl, "CUDA")


@torch.library.register_fake("hpc::fused_speculative_sampler")
def _fused_speculative_sampler_fake(target_logits, draft_token_ids, draft_probs, temperature,
                                    temperature_val, uniform=None, gumbel_noise=None, seed=0):
    B, K = draft_token_ids.shape
    return (target_logits.new_empty((B, K + 1), dtype=torch.int32),
            target_logits.new_empty((B,), dtype=torch.int32))


def fused_speculative_sampler(
    target_logits: Tensor,
    draft_token_ids: Tensor,
    *,
    draft_probs: Optional[Tensor] = None,
    temperature: Union[Tensor, float] = 0.0,
    uniform: Optional[Tensor] = None,
    gumbel_noise: Optional[Tensor] = None,
    seed: int = 0,
) -> Tuple[Tensor, Tensor]:
    """Verify K draft tokens per request against the target model and draw the next token.

    `target_logits` [B * (K + 1), V] (float32 or bfloat16, rows 16-byte aligned, V % 8 == 0,
    V <= 262144): row b * (K + 1) + i is position i of request b, the query order of
    `attention_decode_*` with mtp = K. `draft_token_ids` [B, K] int32 or int64, 1 <= K <= 8.
    Returns `output_token_ids` int32 [B, K + 1] and `num_accepted` int32 [B]: with
    n = num_accepted[b] + 1, out[b, :n] holds the accepted drafts followed by the recovered or bonus
    token, and out[b, n:] is -1. Every written id lies in [0, V).

    With x = float(logits) and ties always going to the smaller token id, request b with
    temperature t (a [B] float32 tensor or one scalar for every request):

    * Greedy (t <= 0 or NaN): a_i = argmax x_i (a row without a non-NaN value gives 0). Draft d_i
      is accepted while d_i == a_i; the first mismatch j emits a_j, and if all K are accepted a_K
      is the bonus token. `draft_probs` is ignored.
    * Sampling (t > 0): xt = x / t (IEEE division), p_i = softmax(xt_i), q_i = draft_probs[b, i]
      ([B, K, V] float32, contiguous) or one-hot at d_i when it is None. d_i is accepted iff
      0 <= d_i < V and u_i * q_i(d_i) < p_i(d_i). At the first rejection j the recovered token is,
      for one-hot drafts, argmax over v != d_j of xt_j + g_j (exactly `fused_sampler` on that row
      with `draft_token_ids=d_j`); with `draft_probs`, argmax over {v : p_j(v) > q_j(v)} of
      log(p_j(v) - q_j(v)) + g_j(v), or argmax of xt_j + g_j when that set is empty. If all K are
      accepted, the bonus token is argmax of xt_K + g_K. So the first emitted token is distributed
      as p whenever the drafts were drawn from q.

    `uniform` [B, K] and `gumbel_noise` [B * (K + 1), V] (float32, contiguous) make the result
    deterministic and must be passed together. Without them the kernels draw Philox4x32-10 noise
    keyed by `seed` (>= 1, needed whenever a request may sample) and the per-stream launch offset
    that `fused_sampler` uses: g of token v in row r from counter (v / 4, r, offset) word v % 4,
    u_{b,i} from counter (0xFFFFFFFF, b * (K + 1) + i, offset) word 0. Each such call advances the
    offset by one, so successive calls and graph replays draw fresh noise.
    """
    t, t_val = _per_row_arg(temperature, "temperature")
    return torch.ops.hpc.fused_speculative_sampler(target_logits, draft_token_ids, draft_probs, t,
                                                   float(t_val), uniform, gumbel_noise, seed)


def _rng_offset(device=None) -> int:
    """Philox launch offset the next internally-seeded sampler call on the current stream of
    `device` will use (synchronises that stream). For tests that reproduce the internal noise."""
    stream = torch.cuda.current_stream(device).cuda_stream
    out = ctypes.c_uint64(0)
    _check_rc(_lib.hpc_sampler_rng_offset(stream, ctypes.byref(out)), "sampler rng offset")
    return out.value
