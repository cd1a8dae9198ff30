"""Time hpc.attention_decode_bf16 (HBM-bound: every K and V element is read once) at the C2 shape in
bf16: batch 64, 32/8 heads, d=128, ~8192 cached tokens per request. GPU box only.

    python tools/decode_bf16_bench.py [--batch 64] [--ctx 8192] [--block 64]

The KV working set (2.1 GB) is far larger than L2; reported = whole call (attention + combine) with
a pre-assigned task map, CUDA events, eager launches.
"""
import argparse
import json
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "hpc-ops_b200"))
import torch  # noqa: E402

import hpc  # noqa: E402
from timing import card, peaks, time_eager  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--ctx", type=int, default=8192)
    ap.add_argument("--hq", type=int, default=32)
    ap.add_argument("--hkv", type=int, default=8)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    dev = "cuda"
    B, hq, hkv, D = a.batch, a.hq, a.hkv, 128
    pk = peaks()
    out = {"card": card(), "batch": B, "ctx": a.ctx, "hq": hq, "hkv": hkv}
    for bs in (64, 16):
        nb = (a.ctx + bs - 1) // bs
        g = torch.Generator(device=dev).manual_seed(0)
        kv = torch.randn(B * nb, 2, bs, hkv, D, device=dev, generator=g).to(torch.bfloat16)
        q = torch.randn(B, hq, D, device=dev, generator=g).to(torch.bfloat16)
        ids = torch.randperm(B * nb, device=dev).to(torch.int32).view(B, nb)
        lens = torch.full((B,), a.ctx, dtype=torch.int32, device=dev)
        tm = hpc.get_attention_decode_task_workspace(B, a.ctx, hkv, 64)
        hpc.assign_attention_decode_task(lens, tm, hkv, 1, True, 64)
        y = torch.empty_like(q)
        fn = lambda: hpc.attention_decode_bf16(q, kv[:, 0], kv[:, 1], ids, lens, new_kv_included=True,  # noqa: E731
                                               task_map=tm, output=y)
        ms = time_eager(fn, a.iters)
        byts = 2 * B * a.ctx * hkv * D * 2 + 2 * B * hq * D * 2
        out[f"block{bs}"] = {"ms": ms, "gbs": byts / ms / 1e6, "frac_hbm": byts / ms / 1e6 / pk["hbm_gbs"],
                             "algorithmic_bytes": byts, "tok_per_s": B / ms * 1e3}
        del kv
    print(json.dumps(out))


if __name__ == "__main__":
    main()
