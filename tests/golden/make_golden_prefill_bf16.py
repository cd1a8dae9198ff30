"""Generate the bf16 prefill fixtures tests/golden/prefill_bf16_*.npz from the REFERENCE's own code,
the way tests/golden/make_golden.py does for the other ops (and with its helpers).

Run in the build container only (needs /root/reference; the GPU box never runs this):
    python tests/golden/make_golden_prefill_bf16.py

The reference keeps its bf16 prefill ground truth as pure-torch functions in its test files; they
are AST-extracted and executed unmodified on CPU, in fp32 on the bf16 inputs.
"""
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent))
from make_golden import OUT, REF, _bf16_bits, extract_many  # noqa: E402

from synth import prefill_bf16 as sp  # noqa: E402  (make_golden put the repository on sys.path)


def dense_case(tag, q_lens, hq, hkv, seed):
    """reference tests/test_attention_prefill_bf16.py `naive_attn_varlen_func` (causal, kv heads
    repeated for GQA)."""
    fn = extract_many(REF / "tests/test_attention_prefill_bf16.py",
                      {"naive_attn_varlen_func"})["naive_attn_varlen_func"]
    d = sp.make_reference_case("dense", q_lens, hq=hq, hkv=hkv, seed=seed)
    g, cu = hq // hkv, d["cu_seqlens_q"]
    gt = fn(d["q"].float(), d["k"].float().repeat_interleave(g, 1),
            d["v"].float().repeat_interleave(g, 1), cu, cu, max(q_lens), max(q_lens), causal=True)
    np.savez_compressed(
        OUT / f"prefill_bf16_{tag}.npz", q=_bf16_bits(d["q"]), k=_bf16_bits(d["k"]),
        v=_bf16_bits(d["v"]), cu_seqlens_q=cu.numpy(), out=gt.float().numpy(),
        meta=np.array([hq, hkv]))
    print("wrote prefill_bf16", tag, gt.shape)


def kvcache_case(tag, num_batch, sq, kv_lens, hq, hkv, page, layout, seed):
    """reference tests/test_attention_with_kvcache_prefill_bf16.py `naive_attn_with_kvcache_func`
    (sq new tokens per request, the last of its kv_lens[b])."""
    fn = extract_many(REF / "tests/test_attention_with_kvcache_prefill_bf16.py",
                      {"naive_attn_with_kvcache_func"})["naive_attn_with_kvcache_func"]
    d = sp.make_reference_case("paged", [sq] * num_batch, kv_lens, hq=hq, hkv=hkv, page=page,
                               layout=layout, seed=seed)
    gt = fn(d["q"].float().reshape(num_batch, sq, hq, 128), d["kcache"].float(),
            d["vcache"].float(), d["seqlens_kv"], d["block_ids"], causal=True)
    np.savez_compressed(
        OUT / f"prefill_bf16_{tag}.npz", q=_bf16_bits(d["q"]), kcache=_bf16_bits(d["kcache"]),
        vcache=_bf16_bits(d["vcache"]), block_ids=d["block_ids"].numpy(),
        seqlens_kv=d["seqlens_kv"].numpy(), cu_seqlens_q=d["cu_seqlens_q"].numpy(),
        out=gt.reshape(-1, hq, 128).float().numpy(),
        meta=np.array([hq, hkv, page, 0 if layout == "NHD" else 1]))
    print("wrote prefill_bf16", tag, gt.shape)


if __name__ == "__main__":
    dense_case("dense", [1, 40, 0, 90], 2, 1, 41)
    kvcache_case("kv_nhd_bs16", 3, 30, [30, 100, 150], 2, 1, 16, "NHD", 42)
    kvcache_case("kv_hnd_bs64", 2, 50, [50, 200], 2, 2, 64, "HND", 43)
