"""Kernel time of the bf16 prefill ops, and torch SDPA (FLASH_ATTENTION backend) on the same dense
inputs, alternated in one run.

    python tools/prefill_bf16_bench.py [--iters 20] [--rounds 5]

Shapes: dense B=1, seq 8192 / 16384 / 32768, GQA 32/8; paged chunked prefill B=4, 2048 new tokens
over 16384 cached, 64-token pages, NHD. Causal FLOP = 4 * 128 * Hq * visible (query, key) pairs;
the share is of the 989 TFLOP/s dense bf16 data-sheet rate of the H100 SXM. SDPA gets K and V
expanded to Hq heads outside the timed region. Prints one JSON line per shape, the card's name,
power limit and max SM clock first.
"""
import argparse
import json
import math
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "hpc-ops_b200"))
import torch  # noqa: E402
from torch.nn.attention import SDPBackend, sdpa_kernel  # noqa: E402

import hpc  # noqa: E402
from synth import prefill_bf16 as sb  # noqa: E402
from timing import BF16_TFLOPS, card, time_eager  # noqa: E402


def pairs(q_lens, kv_lens):
    return sum(q * (kv - q) + q * (q + 1) // 2 for q, kv in zip(q_lens, kv_lens))


def run_shape(name, d, q_lens, kv_lens, args, sdpa=None):
    hq = d["q"].shape[1]

    def ours():
        if d["op"] == "dense":
            return hpc.attention_prefill_bf16(d["q"], d["k"], d["v"], d["seqlens_q"],
                                              d["cu_seqlens_q"], d["max_q"])
        return hpc.attention_with_kvcache_prefill_bf16(d["q"], d["kcache"], d["vcache"],
                                                       d["cu_seqlens_q"], d["block_ids"],
                                                       d["seqlens_kv"], d["max_q"])

    fns = [ours] + ([sdpa] if sdpa else [])
    for f in fns:
        for _ in range(args.warmup):
            f()
    times = [[] for _ in fns]
    for _ in range(args.rounds):
        for i, f in enumerate(fns):
            times[i].append(time_eager(f, args.iters, warm=0))
    med = [sorted(t)[len(t) // 2] for t in times]
    flop = 4 * 128 * hq * pairs(q_lens, kv_lens)
    res = dict(shape=name, ms=round(med[0], 4), tflops=round(flop / med[0] / 1e9, 1),
               share_of_989=round(flop / med[0] / 1e9 / BF16_TFLOPS, 3))
    if sdpa:
        y, ys = ours(), sdpa()
        diff = (y.float() - ys.transpose(0, 1).float()).abs().max()
        res.update(sdpa_flash_ms=round(med[1], 4), sdpa_flash_tflops=round(flop / med[1] / 1e9, 1),
                   speedup_vs_sdpa=round(med[1] / med[0], 3), max_abs_diff_vs_sdpa=float(diff))
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    print(json.dumps({"card": card()}), flush=True)
    hq, hkv = 32, 8
    for seq in (8192, 16384, 32768):
        d = sb.make_reference_case("dense", [seq], hq=hq, hkv=hkv, seed=seq, device="cuda")
        q = d["q"].transpose(0, 1).unsqueeze(0)
        k = d["k"].repeat_interleave(hq // hkv, 1).transpose(0, 1).unsqueeze(0)
        v = d["v"].repeat_interleave(hq // hkv, 1).transpose(0, 1).unsqueeze(0)

        def sdpa():
            with sdpa_kernel(SDPBackend.FLASH_ATTENTION):
                return torch.nn.functional.scaled_dot_product_attention(
                    q, k, v, is_causal=True, scale=1 / math.sqrt(128))[0]

        run_shape(f"dense B=1 seq={seq} Hq={hq} Hkv={hkv}", d, [seq], [seq], args, sdpa)
        del d, q, k, v
    q_lens, kv_lens = [2048] * 4, [16384] * 4
    d = sb.make_reference_case("paged", q_lens, kv_lens, hq=hq, hkv=hkv, page=64, layout="NHD",
                               seed=1, device="cuda")
    run_shape(f"paged B=4 sq=2048 skv=16384 page=64 NHD Hq={hq} Hkv={hkv}", d, q_lens, kv_lens, args)


if __name__ == "__main__":
    main()
