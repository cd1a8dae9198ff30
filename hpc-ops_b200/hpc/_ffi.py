"""ctypes binding of the C-ABI library (include/hpc_b200.h).

The library is the product: if `_C.so` is missing or a launcher reports an error this module
raises — there is no CPU or PyTorch fallback anywhere in `hpc`.
"""
import ctypes
from pathlib import Path

import torch

_pkg_dir = Path(__file__).parent

_so_files = list(_pkg_dir.glob("_C*.so"))
if len(_so_files) != 1:
    raise ImportError(
        f"hpc (H100 build): expected exactly one _C*.so next to {__file__}, found "
        f"{len(_so_files)}. Build it with `python hpc-ops_b200/build.py` (needs nvcc, sm_90a)."
    )
lib = ctypes.CDLL(str(_so_files[0]))

c_int = ctypes.c_int
c_i64 = ctypes.c_int64
c_u32 = ctypes.c_uint32
c_f32 = ctypes.c_float
c_ptr = ctypes.c_void_p

lib.hpc_last_error.restype = ctypes.c_char_p
lib.hpc_version.restype = ctypes.c_char_p
lib.hpc_built_json.restype = ctypes.c_char_p
lib.hpc_sm_count.restype = c_int

lib.hpc_assign_attention_decode_task_host_bytes.restype = c_i64
lib.hpc_assign_attention_decode_task_host_bytes.argtypes = [c_ptr] + [c_int] * 7
lib.hpc_assign_attention_decode_task_sync.restype = c_int
lib.hpc_assign_attention_decode_task_sync.argtypes = [c_ptr] + [c_int] * 7 + [c_ptr, c_i64]
lib.hpc_assign_attention_decode_task_async.restype = c_int
lib.hpc_assign_attention_decode_task_async.argtypes = [c_ptr, c_ptr] + [c_int] * 7 + [c_ptr]

lib.hpc_attention_decode_fp8_async.restype = c_int
lib.hpc_attention_decode_fp8_async.argtypes = (
    [c_ptr] * 13 + [c_int] * 18 + [c_i64] * 6 + [c_ptr]
)

lib.hpc_attention_decode_bf16_async.restype = c_int
lib.hpc_attention_decode_bf16_async.argtypes = [c_ptr] * 10 + [c_int] * 14 + [c_i64] * 6 + [c_ptr]

for _n in ("hpc_attention_decode_fp8_partial_async", "hpc_attention_decode_fp8_combine_async"):
    getattr(lib, _n).restype = c_int
    getattr(lib, _n).argtypes = lib.hpc_attention_decode_fp8_async.argtypes

lib.hpc_group_gemm_blockwise_fp8_async.restype = c_int
lib.hpc_group_gemm_blockwise_fp8_async.argtypes = [c_ptr] * 11 + [c_int] * 10 + [c_ptr]
lib.hpc_group_gemm_fp8_async.restype = c_int
lib.hpc_group_gemm_fp8_async.argtypes = [c_ptr] * 10 + [c_int] * 8 + [c_ptr]
lib.hpc_group_gemm_fp8_multistage_async.restype = c_int
lib.hpc_group_gemm_fp8_multistage_async.argtypes = [c_ptr] * 9 + [c_int] * 7 + [c_ptr]
lib.hpc_group_gemm_fp8_scatter_async.restype = c_int
lib.hpc_group_gemm_fp8_scatter_async.argtypes = [c_ptr] * 10 + [c_int] * 7 + [c_ptr, c_int, c_ptr]
lib.hpc_act_mul_and_quant_async.restype = c_int
lib.hpc_act_mul_and_quant_async.argtypes = [c_ptr] * 3 + [c_int] * 3 + [c_ptr]
lib.hpc_scaled_fp8_quant_async.restype = c_int
lib.hpc_scaled_fp8_quant_async.argtypes = [c_ptr] * 3 + [c_i64, c_int, c_ptr]
lib.hpc_reformat_x_scale_async.restype = c_int
lib.hpc_reformat_x_scale_async.argtypes = [c_ptr] * 4 + [c_int] * 4 + [c_ptr]
lib.hpc_count_and_gather_async.restype = c_int
lib.hpc_count_and_gather_async.argtypes = [c_ptr] * 15 + [c_int] * 7 + [c_ptr]
lib.hpc_blockwise_count_and_gather_async.restype = c_int
lib.hpc_blockwise_count_and_gather_async.argtypes = [c_ptr] * 17 + [c_int] * 9 + [c_ptr]
lib.hpc_reduce_async.restype = c_int
lib.hpc_reduce_async.argtypes = [c_ptr] * 5 + [c_int] * 5 + [c_ptr]
lib.hpc_fuse_moe_async.restype = c_int
lib.hpc_fuse_moe_async.argtypes = [c_ptr] * 23 + [c_int] * 10 + [c_ptr]
lib.hpc_fuse_moe_blockwise_async.restype = c_int
lib.hpc_fuse_moe_blockwise_async.argtypes = [c_ptr] * 25 + [c_int] * 12 + [c_ptr]

lib.hpc_fuse_allreduce_rmsnorm_high_throughput_async.restype = c_int
lib.hpc_fuse_allreduce_rmsnorm_high_throughput_async.argtypes = (
    [c_ptr] * 8 + [c_i64] * 3 + [ctypes.c_double, c_int, c_int, c_ptr])
lib.hpc_fuse_allreduce_rmsnorm_high_throughput_p2p_async.restype = c_int
lib.hpc_fuse_allreduce_rmsnorm_high_throughput_p2p_async.argtypes = (
    [c_ptr] * 10 + [c_i64] * 3 + [ctypes.c_double, c_int, c_int, c_ptr])
lib.hpc_fuse_allreduce_rmsnorm_low_latency_async.restype = c_int
lib.hpc_fuse_allreduce_rmsnorm_low_latency_async.argtypes = (
    [c_int] * 4 + [c_ptr] * 4 + [c_int] * 2 + [c_ptr] * 3 + [ctypes.c_double] + [c_ptr] * 2 + [c_int, c_ptr])
lib.hpc_fuse_allreduce_rmsnorm_low_latency_ex_async.restype = c_int
lib.hpc_fuse_allreduce_rmsnorm_low_latency_ex_async.argtypes = (
    [c_int] * 4 + [c_ptr] * 4 + [c_int] * 2 + [c_ptr] * 3 + [ctypes.c_double] + [c_ptr] * 2 + [c_int, c_int, c_ptr])

lib.hpc_gemm_bf16xfp32_select_splitk.restype = c_int
lib.hpc_gemm_bf16xfp32_select_splitk.argtypes = [c_int] * 4
lib.hpc_gemm_bf16xfp32_async.restype = c_int
lib.hpc_gemm_bf16xfp32_async.argtypes = [c_ptr] * 6 + [c_int] * 3 + [c_f32] + [c_int] * 5 + [c_ptr]

_prefill_args = [c_ptr] * 11 + [c_int] * 14 + [c_i64] * 6
lib.hpc_attention_blocksparse_prefill_qpertoken_perhead_kvpertensor_fp8_async.restype = c_int
lib.hpc_attention_blocksparse_prefill_qpertoken_perhead_kvpertensor_fp8_async.argtypes = (
    _prefill_args + [c_ptr])
lib.hpc_attention_blocksparse_prefill_qkpertoken_perhead_vperhead_fp8_async.restype = c_int
lib.hpc_attention_blocksparse_prefill_qkpertoken_perhead_vperhead_fp8_async.argtypes = (
    _prefill_args + [c_i64] * 3 + [c_ptr])

# (hasattr: a library built from an older commit, e.g. for an A/B timing, lacks these symbols; it
# still fails loudly -- at the first rope, sampler, speculative sampler, bf16 prefill, Stem, RMSNorm
# or masked activation call)
if hasattr(lib, "hpc_rope_norm_store_kv_async"):
    lib.hpc_rope_norm_store_kv_async.restype = c_int
    lib.hpc_rope_norm_store_kv_async.argtypes = [c_ptr] * 12 + [c_int] * 12 + [c_ptr]
    lib.hpc_rope_norm_store_kv_fp8_async.restype = c_int
    lib.hpc_rope_norm_store_kv_fp8_async.argtypes = [c_ptr] * 17 + [c_f32] + [c_int] * 14 + [c_ptr]

if hasattr(lib, "hpc_attention_prefill_bf16_async"):
    lib.hpc_attention_prefill_bf16_async.restype = c_int
    lib.hpc_attention_prefill_bf16_async.argtypes = [c_ptr] * 6 + [c_int] * 11 + [c_ptr]
    lib.hpc_attention_with_kvcache_prefill_bf16_async.restype = c_int
    lib.hpc_attention_with_kvcache_prefill_bf16_async.argtypes = (
        [c_ptr] * 7 + [c_int] * 12 + [c_i64] * 6 + [c_ptr])

if hasattr(lib, "hpc_fused_sampler_async"):
    lib.hpc_fused_sampler_async.restype = c_int
    lib.hpc_fused_sampler_async.argtypes = (
        [c_ptr, c_ptr, c_i64, c_int, c_int, c_int, c_ptr, c_i64, c_ptr, c_ptr, c_f32, c_ptr, c_f32,
         c_int, c_ptr, c_int, c_int, c_ptr, c_f32, c_int, c_ptr, ctypes.c_uint64, c_ptr])
    lib.hpc_fused_sampler_temperature_sample_async.restype = c_int
    lib.hpc_fused_sampler_temperature_sample_async.argtypes = (
        [c_ptr, c_ptr, c_i64, c_int, c_int, c_int, c_ptr, c_f32, c_ptr, c_ptr, ctypes.c_uint64, c_ptr])
    lib.hpc_sampler_rng_offset.restype = c_int
    lib.hpc_sampler_rng_offset.argtypes = [c_ptr, ctypes.POINTER(ctypes.c_uint64)]

if hasattr(lib, "hpc_fused_speculative_sampler_async"):
    lib.hpc_fused_speculative_sampler_async.restype = c_int
    lib.hpc_fused_speculative_sampler_async.argtypes = (
        [c_ptr] * 4 + [c_i64] + [c_int] * 4 + [c_ptr, c_int, c_ptr, c_ptr, c_f32, c_ptr, c_ptr,
                                              ctypes.c_uint64, c_ptr])

if hasattr(lib, "hpc_stem_tpd_async"):
    lib.hpc_stem_oam_prep_paged_kv_qpertoken_perhead_kvpertensor_dim128_async.restype = c_int
    lib.hpc_stem_oam_prep_paged_kv_qpertoken_perhead_kvpertensor_dim128_async.argtypes = (
        [c_ptr] * 8 + [c_int] * 9 + [c_f32, c_int, c_int] + [c_i64] * 6 + [c_ptr, c_ptr])
    lib.hpc_stem_oam_prep_paged_kv_qkpertoken_perhead_vperhead_dim128_async.restype = c_int
    lib.hpc_stem_oam_prep_paged_kv_qkpertoken_perhead_vperhead_dim128_async.argtypes = (
        [c_ptr] * 8 + [c_int] * 10 + [c_f32, c_int, c_int] + [c_i64] * 9 + [c_ptr, c_ptr])
    lib.hpc_stem_oam_prep_varlen_q_dim128_async.restype = c_int
    lib.hpc_stem_oam_prep_varlen_q_dim128_async.argtypes = (
        [c_ptr] * 5 + [c_int] * 6 + [c_i64] * 3 + [c_ptr])
    lib.hpc_stem_oam_gemm_dim128_async.restype = c_int
    lib.hpc_stem_oam_gemm_dim128_async.argtypes = [c_ptr] * 6 + [c_int] * 8 + [c_ptr]
    lib.hpc_stem_tpd_async.restype = c_int
    lib.hpc_stem_tpd_async.argtypes = (
        [c_ptr] * 5 + [c_int] * 5 + [c_f32, c_int, c_int, c_f32, c_int, c_f32, c_int, c_ptr])


if hasattr(lib, "hpc_fused_rmsnorm_with_scale_async"):
    lib.hpc_fused_rmsnorm_with_scale_async.restype = c_int
    lib.hpc_fused_rmsnorm_with_scale_async.argtypes = [c_ptr] * 6 + [c_f32] + [c_int] * 3 + [c_ptr]
    lib.hpc_masked_act_mul_and_quant_async.restype = c_int
    lib.hpc_masked_act_mul_and_quant_async.argtypes = [c_ptr] * 4 + [c_int] * 3 + [c_ptr]
    lib.hpc_masked_act_mul_and_blockwise_quant_async.restype = c_int
    lib.hpc_masked_act_mul_and_blockwise_quant_async.argtypes = [c_ptr] * 4 + [c_int] * 3 + [c_ptr]

if hasattr(lib, "hpc_moe_topk_gating_async"):
    lib.hpc_moe_topk_gating_async.restype = c_int
    lib.hpc_moe_topk_gating_async.argtypes = [c_ptr] * 4 + [c_int] * 8 + [c_i64, c_f32, c_ptr]

def check(rc: int, what: str = ""):
    """Turn a launcher status into the RuntimeError the reference raises via TORCH_CHECK."""
    if rc != 0:
        msg = lib.hpc_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"hpc {what} failed (code {rc}): {msg}")


def ptr(t):
    """Raw data pointer of a tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def stream_of(t) -> int:
    """cudaStream_t of torch's current stream on the tensor's device."""
    return torch.cuda.current_stream(t.device).cuda_stream


_sm_count_cache = {}


def sm_count(device=None) -> int:
    dev = torch.cuda.current_device() if device is None else torch.device(device).index
    if dev is None:
        dev = torch.cuda.current_device()
    if dev not in _sm_count_cache:
        _sm_count_cache[dev] = torch.cuda.get_device_properties(dev).multi_processor_count
    return _sm_count_cache[dev]
