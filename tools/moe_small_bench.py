"""Decode-regime FusedMoE (per-tensor FP8) at the reference's small-M shape
(tests/test_fuse_moe_cp_async.py:147-156: T=128, E=128, top-8, H=4096, I=192 — the shape its cp.async
path exists for): time vs the HBM floor of streaming the touched expert weights once. GPU box only.

    python tools/moe_small_bench.py [--tokens 128] [--inter 192]
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
from timing import card, peaks, time_graph  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=128)
    ap.add_argument("--experts", type=int, default=128)
    ap.add_argument("--topk", type=int, default=8)
    ap.add_argument("--hidden", type=int, default=4096)
    ap.add_argument("--inter", type=int, default=192)
    a = ap.parse_args()
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(41)
    T, E, K, H, I = a.tokens, a.experts, a.topk, a.hidden, a.inter
    ids = torch.multinomial(torch.ones((T, E), device=dev), K, generator=g).to(torch.int32)
    ids, _ = torch.sort(ids, dim=1)
    ts = torch.rand((T, K), generator=g, device=dev)
    x = torch.randn((T, H), generator=g, device=dev).to(torch.float8_e4m3fn)
    guw = torch.randn((E, 2 * I, H), generator=g, device=dev).to(torch.float8_e4m3fn)
    dw = torch.randn((E, H, I), generator=g, device=dev).to(torch.float8_e4m3fn)
    gus = torch.rand((E,), generator=g, device=dev) * 0.01
    ds = torch.rand((E,), generator=g, device=dev) * 0.01
    acts = torch.rand((1,), generator=g, device=dev) + 0.5

    def run():
        return hpc.fuse_moe(x, guw, dw, gus, ds, acts, ids, ts, 0, E, use_bf16_mul=True)

    y = run()
    torch.cuda.synchronize()
    assert torch.isfinite(y.float()).all()
    ms = time_graph(run, reps=10, iters=5)
    touched = int(torch.unique(ids).numel())
    wbytes = touched * 3 * I * H
    pk = peaks()
    print(json.dumps({"card": card(), "us": ms * 1e3, "experts_touched": touched,
                      "rows_per_expert_avg": T * K / E, "weight_bytes": wbytes, "hbm_floor_us": wbytes / pk["hbm_gbs"] / 1e3,
                      "frac_of_hbm_floor": (wbytes / pk["hbm_gbs"] / 1e3) / (ms * 1e3),
                      "tok_per_s": T / ms * 1e3, "cfg": vars(a),
                      "timing": "CUDA-graph replay, 10 calls per graph x 5 replays"}))


if __name__ == "__main__":
    main()
