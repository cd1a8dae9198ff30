"""Fused speculative sampler benchmark: CUDA-graph replays of hpc.fused_speculative_sampler against
the same verification written as torch ops (synth/spec_sampler.py's vLLM-style chain, drawing its
noise with torch), bf16 logits.

    python tools/spec_sampler_bench.py [--vocab 120832,151936] [--batches 1,8,64,256] [--k 1,3] [--json PATH]

Per shape (V, B, K, one-hot or draft_probs) and noise (drawn in the kernel or given): µs per call
(median of 5 windows of graph replays, with the min-max), the floor B (K + 1) V esz + B V esz
(+ B V 4 with draft_probs) at the data-sheet HBM bandwidth and the call's share of it, and the
torch chain's µs. Kernel times of the two passes come from torch.profiler in a separate run of
eager calls, with pass 1's share of HBM bandwidth for its B (K + 1) V esz bytes. Every request
samples (t = 0.8). GPU only.
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
from synth.spec_sampler import torch_chain  # noqa: E402
from timing import card, peaks, spread, time_graph  # noqa: E402

T = 0.8


def inputs(B, K, V, probs):
    g = torch.Generator(device="cpu").manual_seed(B * 100 + K)
    logits = (torch.randn(B * (K + 1), V, generator=g) * 2).to(torch.bfloat16).cuda()
    draft = torch.randint(0, V, (B, K), generator=g).cuda()
    q = None
    if probs:
        q = torch.softmax(torch.randn(B, K, V, generator=g) * 2, -1).cuda()
    u = torch.rand(B, K, device="cuda")
    noise = -(-torch.rand(B * (K + 1), V, device="cuda").clamp_(2.0 ** -24, 1 - 2.0 ** -24).log()).log()
    return logits, draft, q, u, noise


def kernel_us(fn, calls=10):
    """Mean device time per call of each spec_* kernel, from torch.profiler."""
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for name in ("spec_row_stats_kernel", "spec_sample_kernel"):
            if name in e.key:
                out[name] = round(e.device_time_total / calls, 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vocab", default="120832,151936")
    ap.add_argument("--batches", default="1,8,64,256")
    ap.add_argument("--k", default="1,3")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "spec_sampler_bench needs a GPU"
    gpu = card()
    hbm = peaks()["hbm_gbs"] * 1e9
    rows = []
    for V in [int(v) for v in a.vocab.split(",")]:
        for B in [int(b) for b in a.batches.split(",")]:
            for K in [int(k) for k in a.k.split(",")]:
                for probs in (False, True):
                    logits, draft, q, u, noise = inputs(B, K, V, probs)
                    temp = torch.full((B,), T, device="cuda")
                    floor = B * (K + 1) * V * 2 + B * V * 2 + (B * V * 4 if probs else 0)

                    def chain():
                        uu = torch.rand(B, K, device="cuda")
                        gg = -(-torch.rand(B * (K + 1), V, device="cuda").clamp_(2.0 ** -24, 1 - 2.0 ** -24)
                               .log()).log()
                        return torch_chain(logits, draft, q, temp, uu, gg)

                    scenes = {
                        "internal": lambda: hpc.fused_speculative_sampler(logits, draft, draft_probs=q,
                                                                          temperature=T, seed=7),
                        "given": lambda: hpc.fused_speculative_sampler(logits, draft, draft_probs=q, temperature=T,
                                                                       uniform=u, gumbel_noise=noise),
                    }
                    torch_ms = spread(lambda: time_graph(chain, reps=10, iters=5), 5)
                    for name, fn in scenes.items():
                        ms = spread(lambda: time_graph(fn, reps=20, iters=10), 5)
                        k = kernel_us(fn)
                        p1 = k.get("spec_row_stats_kernel")
                        rows.append(dict(
                            V=V, B=B, K=K, drafts="probs" if probs else "onehot", noise=name,
                            us=round(ms[0] * 1e3, 2), us_min=round(ms[1] * 1e3, 2), us_max=round(ms[2] * 1e3, 2),
                            floor_us=round(floor / hbm * 1e6, 2), hbm_share=round(floor / (ms[0] * 1e-3) / hbm, 3),
                            pass1_us=p1, pass2_us=k.get("spec_sample_kernel"),
                            pass1_hbm_share=round(B * (K + 1) * V * 2 / (p1 * 1e-6) / hbm, 3) if p1 else None,
                            torch_us=round(torch_ms[0] * 1e3, 2), speedup=round(torch_ms[0] / ms[0], 2)))
                        print(json.dumps(rows[-1]), flush=True)
                    del logits, draft, q, u, noise
                    torch.cuda.empty_cache()
    res = dict(card=gpu, hbm_gbs=hbm / 1e9, rows=rows)
    if a.json:
        Path(a.json).parent.mkdir(parents=True, exist_ok=True)
        Path(a.json).write_text(json.dumps(res, indent=1))
    print(json.dumps(dict(card=gpu)))


if __name__ == "__main__":
    main()
