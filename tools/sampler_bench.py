"""Fused sampler benchmark: CUDA-graph replays of hpc.fused_sampler at V = 120832, bf16 logits.

    python tools/sampler_bench.py [--batches 1,8,16,32,64,128,256,512] [--out PATH]

Scenes (the reference benchmark's defaults): `temperature` (T = 0.7, internal noise) and `full`
(repetition penalty 1.05, T = 0.7, top-k 20, top-p 0.9, AFTER_TOPK, internal noise); and
`temperature_given_noise`, the first with a float32 noise tensor passed in, to separate the cost of
drawing noise in the kernel from the cost of streaming the logits. Per point: µs per
call, the bytes the call must move (from the shapes), their share of the 3.35 TB/s data-sheet HBM
bandwidth, and the same sampling written as a chain of torch ops, timed the same way in this process.
GPU only.
"""
import argparse
import json
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "hpc-ops_b200"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import hpc  # noqa: E402
from timing import card, peaks, time_graph  # noqa: E402

V = 120832
T, RP, TOPK, TOPP = 0.7, 1.05, 20, 0.9


def inputs(B):
    g = torch.Generator(device="cpu").manual_seed(B)
    logits = torch.randn(B, V, generator=g).to(torch.bfloat16).cuda()
    seen = torch.rand(B, V, generator=g) < 0.002  # ~240 previously generated tokens per row
    mask = torch.from_numpy(np.packbits(seen.numpy(), axis=-1, bitorder="little")).cuda()
    return logits, mask, seen.cuda(), torch.arange(B, dtype=torch.int32, device="cuda")


def torch_temperature(logits):
    probs = (logits.float() / T).softmax(-1)
    return (probs / torch.empty_like(probs).exponential_()).argmax(-1, keepdim=True).int()


def torch_full(logits, seen):
    x = logits.float()
    x = torch.where(seen, torch.where(x > 0, x / RP, x * RP), x) / T
    val, idx = x.topk(TOPK, -1)
    p = val.softmax(-1)
    excl = p.cumsum(-1) - p
    p = p.masked_fill(excl >= TOPP, 0)
    pick = (p / torch.empty_like(p).exponential_()).argmax(-1, keepdim=True)
    tok = idx.gather(-1, pick)
    return tok.int()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,16,32,64,128,256,512")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "sampler_bench needs a GPU"
    gpu = card()
    hbm = peaks()["hbm_gbs"]
    rows = []
    for B in [int(b) for b in a.batches.split(",")]:
        logits, mask, seen, slot = inputs(B)
        rp = torch.full((B,), RP, device="cuda")
        u = torch.rand(B, V, device="cuda").clamp_(2.0 ** -24, 1 - 2.0 ** -24)
        noise = -(-u.log()).log()
        scenes = {
            "temperature": (lambda: hpc.fused_sampler(logits, temperature=T, seed=7),
                            lambda: torch_temperature(logits), B * V * 2 + B * 4),
            "full": (lambda: hpc.fused_sampler(logits, penalty_mask=mask, slot_id=slot, repetition_penalty=rp,
                                               temperature=T, softmax_policy=hpc.SoftmaxPolicy.AFTER_TOPK,
                                               topk=TOPK, topp=TOPP, max_topk=32, seed=7),
                     lambda: torch_full(logits, seen), B * V * 2 + B * V // 8 + B * 16),
            # the temperature scene with the noise passed in: 3x the bytes, no Philox or logf in the
            # kernel; against `temperature` it shows what drawing the noise costs
            "temperature_given_noise": (lambda: hpc.fused_sampler(logits, temperature=T, gumbel_noise=noise),
                                        lambda: ((logits.float() / T) + noise).argmax(-1, keepdim=True).int(),
                                        B * V * 6 + B * 4),
        }
        for name, (ours, ref, nbytes) in scenes.items():
            ms = time_graph(ours, reps=20, iters=20)
            ms_torch = time_graph(ref, reps=20, iters=20)
            rows.append(dict(scene=name, batch=B, us=round(ms * 1e3, 2), bytes=nbytes,
                             hbm_share=round(nbytes / (ms * 1e-3) / (hbm * 1e9), 3),
                             torch_us=round(ms_torch * 1e3, 2), speedup=round(ms_torch / ms, 2)))
            print(json.dumps(rows[-1]), flush=True)
    res = dict(card=gpu, vocab=V, hbm_gbs=hbm, rows=rows)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))
    print(json.dumps(dict(card=gpu)))


if __name__ == "__main__":
    main()
