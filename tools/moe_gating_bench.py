"""Time MoE top-k gating (hpc.moe_topk_gating) against the same computation written as an fp32 torch
chain (synth/moe_gating.py: softmax / sigmoid -> grouped mask -> topk -> gather -> renormalize):

    python tools/moe_gating_bench.py [--iters 50] [--reps 5] [--json out.json]

Every figure is the time of one call from CUDA events around `iters` replays of a CUDA graph
holding that call, the median (and min, max) of `reps` warmed windows. The torch chain is captured
and timed the same way, and so is a one-element torch add, the cost of one kernel launch from a
graph. For each shape: the bytes the call must move (logits, bias, ids and weights) and their
share of the H100 SXM data-sheet 3.35 TB/s. The card's name, power limit and max SM clock are read
in the same run.

Shapes: fp32 logits at T in {1, 16, 128, 1024, 4096, 16384, 65536} for the Qwen3 (128 experts,
softmax, top-8), DeepSeek-V3 (256, sigmoid + bias, 8 groups, top-4 groups, top-8) and Qwen3-Next
(512, softmax, top-10) routers."""
import argparse
import json
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "hpc-ops_b200"))
import torch  # noqa: E402

import hpc  # noqa: E402
from synth import moe_gating as sg  # noqa: E402
from timing import HBM_GBS, card, spread, time_graph  # noqa: E402

HBM = HBM_GBS * 1e9
FAMILIES = ("qwen3", "deepseek_v3", "qwen3_next")
TOKENS = (1, 16, 128, 1024, 4096, 16384, 65536)


def graphed_us(fn, a):
    """Median, min and max in µs of `a.reps` windows of `a.iters` replays of a graph of one call."""
    return [t * 1e3 for t in spread(lambda: time_graph(fn, 1, a.iters), a.reps)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    res = {"card": card(), "rows": []}
    z = torch.zeros(1, device="cuda")
    launch = graphed_us(lambda: z.add_(1), a)
    res["one_launch_us"] = [round(v, 2) for v in launch]
    print(json.dumps({"card": res["card"], "one_launch_us": res["one_launch_us"]}), flush=True)
    for name in FAMILIES:
        cfg = sg.CONFIGS[name]
        E, k = cfg["E"], cfg["topk"]
        bias = (torch.randn(E, device="cuda") * 0.1) if cfg["bias"] else None
        kw = sg.hpc_kwargs(cfg, bias)
        for T in TOKENS:
            x = sg.random_logits(T, E, seed=T, device="cuda")
            ids, w = hpc.moe_topk_gating(x, **kw)
            tids, tw = sg.torch_chain(x, **kw)
            same = bool(torch.equal(ids, tids))
            ours = graphed_us(lambda: hpc.moe_topk_gating(x, **kw), a)
            ref = graphed_us(lambda: sg.torch_chain(x, **kw), a)
            by = T * E * 4 + (E * 4 if bias is not None else 0) + T * k * 8
            t = ours[0]
            r = dict(family=name, T=T, E=E, topk=k, us=round(t, 2), us_min=round(ours[1], 2),
                     us_max=round(ours[2], 2), bytes=by, hbm_share=round(by / HBM * 1e6 / t, 3),
                     torch_us=[round(v, 2) for v in ref], speedup=round(ref[0] / t, 2),
                     launches=round(t / launch[0], 2), ids_equal_torch=same)
            print(json.dumps(r), flush=True)
            res["rows"].append(r)
    if a.json:
        Path(a.json).parent.mkdir(parents=True, exist_ok=True)
        Path(a.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
