"""Time the FusedMoE blockwise pipeline at BASELINE config C3, or another shape, with the sampled
oracle parity check of bench.py's `moe_c3` entry (tools/bench_extras.py). Needs a GPU.

    python tools/moe_bench.py [--tokens 4096] [--experts 128] [--topk 8] [--hidden 4096] [--inter 14336]
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
    ap.add_argument("--tokens", type=int, default=4096)
    ap.add_argument("--experts", type=int, default=128)
    ap.add_argument("--topk", type=int, default=8)
    ap.add_argument("--hidden", type=int, default=4096)
    ap.add_argument("--inter", type=int, default=14336)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    cfg = dict(tokens=a.tokens, topk=a.topk, experts=a.experts, hidden=a.hidden, inter=a.inter)
    res = bx.moe_c3(hpc, torch.device("cuda", 0), a.iters, parity_tokens=(a.tokens - 1,), cfg=cfg)
    print(json.dumps({"card": card(), **res}))


if __name__ == "__main__":
    main()
