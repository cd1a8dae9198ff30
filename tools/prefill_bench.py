"""Time the FP8 block-sparse prefill at BASELINE config C4 (B=1, seq=32768, GQA 32/8, d=128,
25 % of causal 128x128 tiles + diagonal), or another shape, with the sampled oracle parity check of
bench.py's `prefill_c4_*` entries (tools/bench_extras.py). Needs a GPU.

    python tools/prefill_bench.py [--seq 32768] [--skip 0.75] [--kpt 1]
"""
import argparse
import json
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "hpc-ops_b200"))
import torch  # noqa: E402

import bench_extras as bx  # noqa: E402
import hpc  # noqa: E402
from timing import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq", type=int, default=32768)
    ap.add_argument("--hq", type=int, default=32)
    ap.add_argument("--hkv", type=int, default=8)
    ap.add_argument("--skip", type=float, default=0.75)
    ap.add_argument("--kpt", type=int, default=1)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    cfg = dict(seq=a.seq, hq=a.hq, hkv=a.hkv, skip=a.skip)
    res = bx.prefill_c4(hpc, torch.device("cuda", 0), bool(a.kpt), a.iters, cfg=cfg)
    print(json.dumps({"card": card(), **res}))


if __name__ == "__main__":
    main()
