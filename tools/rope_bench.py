"""Time hpc.rope_norm_store_kv_fp8 / rope_norm_store_kv (HBM-bound streaming kernel) against the
measured copy bandwidth. GPU box only.

    python tools/rope_bench.py [--rows 32768] [--hq 32] [--hkv 8]
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
    ap.add_argument("--rows", type=int, default=32768, help="prefill tokens of one request")
    ap.add_argument("--hq", type=int, default=32)
    ap.add_argument("--hkv", type=int, default=8)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    dev = "cuda"
    D, bs = 128, 64
    T, hq, hkv = a.rows, a.hq, a.hkv
    g = torch.Generator(device=dev).manual_seed(0)
    qkv = torch.randn(T, (hq + 2 * hkv) * D, device=dev, generator=g).to(torch.bfloat16)
    nblk = (T + bs - 1) // bs
    from synth.rope import generate_cos_sin_cache
    cos_sin = generate_cos_sin_cache(T, D).to(dev)
    seqlen = torch.tensor([T], dtype=torch.int32, device=dev)
    q_index = torch.tensor([0, T], dtype=torch.int32, device=dev)
    kv_idx = torch.randperm(nblk, device=dev).to(torch.int32).view(1, -1)
    ks = torch.tensor([0.1], device=dev)
    vs = torch.tensor([0.1], device=dev)
    pk = peaks()
    res = {}
    for name, fp8 in (("bf16", False), ("fp8_dynamic_q", True)):
        dt = torch.float8_e4m3fn if fp8 else torch.bfloat16
        kc = torch.zeros(nblk, bs, hkv, D, device=dev, dtype=torch.bfloat16).to(dt)
        vc = torch.zeros(nblk, bs, hkv, D, device=dev, dtype=torch.bfloat16).to(dt)
        if fp8:
            fn = lambda: hpc.rope_norm_store_kv_fp8(kc, vc, qkv, cos_sin, seqlen, q_index, kv_idx, True,  # noqa: E731
                                                    ks, vs, 1, max_seqlens=T)
        else:
            fn = lambda: hpc.rope_norm_store_kv(kc, vc, qkv, cos_sin, seqlen, q_index, kv_idx, True)  # noqa: E731
        ms = time_eager(fn, a.iters)
        ob = 1 if fp8 else 2
        byts = T * (hq + 2 * hkv) * D * 2 + T * (hq + 2 * hkv) * D * ob + T * D * 4 + (T * hq * 4 if fp8 else 0)
        res[name] = {"ms": ms, "gbs": byts / ms / 1e6, "frac_hbm": byts / ms / 1e6 / pk["hbm_gbs"],
                     "algorithmic_bytes": byts, "tok_per_s": T / ms * 1e3}
    print(json.dumps({"card": card(), "rows": T, "hq": hq, "hkv": hkv, **res}))


if __name__ == "__main__":
    main()
