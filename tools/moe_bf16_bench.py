"""Time the bf16 FusedMoE (hpc.fuse_moe_bf16) against the same layer written in torch (gather ->
torch._grouped_mm -> silu * mul -> torch._grouped_mm -> weighted sum, or a per-expert matmul loop
where torch._grouped_mm rejects the shape):

    python tools/moe_bf16_bench.py [--iters 5] [--reps 3] [--json out.json]

Every figure is the time of one call from CUDA events around `iters` replays of a CUDA graph
holding 5 calls, the median (and min, max) of `reps` warmed windows; the torch chain is captured
and timed the same way (eagerly, and marked so, if it cannot be captured). Per call: the FLOPs
2 * rows * 3 * H * I, the bytes it must move (the weights of the experts that received rows, x and
y) and the least time the H100 SXM data sheet allows for them (989 TFLOP/s bf16, 3.35 TB/s), named
by the bound that sets it, as a share of the measured time. The card's name, power limit and SM
clocks are read in the same run.

Shapes: Qwen3-30B-A3B-like (128 experts, top-8, H 2048, I 768) and Mixtral-like (8 experts, top-2,
H 4096, I 14336) at T in {1, 64, 512, 4096, 16384}, uniform routing."""
import argparse
import json
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "hpc-ops_b200"))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import hpc  # noqa: E402
from timing import BF16_TFLOPS, HBM_GBS, card, spread, time_eager, time_graph  # noqa: E402

SHAPES = {"qwen3_30b_a3b": (128, 8, 2048, 768), "mixtral_8x7b": (8, 2, 4096, 14336)}
TOKENS = (1, 64, 512, 4096, 16384)


def make(E, k, H, I, T, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((T, H), generator=g, device="cuda").to(torch.bfloat16)
    guw = (torch.randn((E, 2 * I, H), generator=g, device="cuda") * (2 / H ** 0.5)).to(torch.bfloat16)
    dw = (torch.randn((E, H, I), generator=g, device="cuda") / (1.5 * I ** 0.5)).to(torch.bfloat16)
    ids = torch.rand((T, E), generator=g, device="cuda").topk(k, dim=1).indices.to(torch.int32)
    w = torch.rand((T, k), generator=g, device="cuda") + 0.1
    return x, guw, dw, ids.contiguous(), (w / w.sum(1, keepdim=True)).contiguous()


def torch_layer(x, guw, dw, ids, w, grouped):
    """The layer in torch, no host synchronisation (capturable)."""
    T, H = x.shape
    E, I2, _ = guw.shape
    flat = ids.reshape(-1).long()
    order = torch.argsort(flat, stable=True)
    xs = x[order // ids.size(1)]
    if grouped:
        counts = torch.zeros(E, dtype=torch.int32, device=x.device).scatter_add_(
            0, flat, torch.ones_like(flat, dtype=torch.int32))
        offs = torch.cumsum(counts, 0, dtype=torch.int32)
        gu = torch._grouped_mm(xs, guw.transpose(1, 2), offs=offs)
        a = F.silu(gu[:, :I2 // 2]) * gu[:, I2 // 2:]
        d = torch._grouped_mm(a, dw.transpose(1, 2), offs=offs)
    else:
        sorted_ids = flat[order]
        d = torch.empty((xs.size(0), H), dtype=x.dtype, device=x.device)
        for e in range(E):
            sel = sorted_ids == e
            gu = xs[sel] @ guw[e].t()
            d[sel] = (F.silu(gu[:, :I2 // 2]) * gu[:, I2 // 2:]) @ dw[e].t()
    out = torch.empty_like(d)
    out[order] = d
    return (out.view(T, -1, H).float() * w[..., None]).sum(1).to(torch.bfloat16)


def timed_us(fn, a):
    """(median, min, max) µs per call and how it was timed."""
    try:
        return [t * 1e3 for t in spread(lambda: time_graph(fn, 5, a.iters), a.reps)], "graph"
    except Exception:  # noqa: BLE001 - a torch op that cannot be captured is timed eagerly
        torch.cuda.synchronize()
        return [t * 1e3 for t in spread(lambda: time_eager(fn, 5 * a.iters), a.reps)], "eager"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    res = {"card": card(), "rows": []}
    print(json.dumps({"card": res["card"]}), flush=True)
    for name, (E, k, H, I) in SHAPES.items():
        for T in TOKENS:
            x, guw, dw, ids, w = make(E, k, H, I, T, seed=T)
            fn = lambda: hpc.fuse_moe_bf16(x, guw, dw, ids, w, 0, E)  # noqa: E731
            y = fn()
            grouped = True
            try:
                ref = torch_layer(x, guw, dw, ids, w, True)
            except Exception:  # noqa: BLE001 - torch._grouped_mm rejects the shape
                grouped = False
                ref = torch_layer(x, guw, dw, ids, w, False)
            torch.cuda.synchronize()
            rel = float((y.float() - ref.float()).norm() / ref.float().norm())
            ours, _ = timed_us(fn, a)
            base, how = timed_us(lambda: torch_layer(x, guw, dw, ids, w, grouped), a)
            used = int((torch.bincount(ids.reshape(-1).long(), minlength=E) > 0).sum())
            rows = T * k
            flops = 2.0 * rows * 3 * H * I
            nbytes = used * 3 * H * I * 2 + 2 * T * H * 2
            t_flop, t_byte = flops / (BF16_TFLOPS * 1e12), nbytes / (HBM_GBS * 1e9)
            roof_us = max(t_flop, t_byte) * 1e6
            row = dict(shape=name, T=T, us=[round(v, 2) for v in ours],
                       torch_us=[round(v, 2) for v in base],
                       torch=("_grouped_mm" if grouped else "matmul loop") + f" ({how})",
                       speedup=round(base[0] / ours[0], 2), rel_err_vs_torch=round(rel, 5),
                       experts_used=used, gflop=round(flops / 1e9, 2), mbytes=round(nbytes / 1e6, 1),
                       bound="compute" if t_flop > t_byte else "HBM",
                       share_of_roof=round(roof_us / ours[0], 3),
                       tflops=round(flops / ours[0] / 1e6, 1), gbs=round(nbytes / ours[0] / 1e3, 1))
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
            del x, guw, dw, ids, w, y, ref
            torch.cuda.empty_cache()
    if a.json:
        Path(a.json).parent.mkdir(parents=True, exist_ok=True)
        Path(a.json).write_text(json.dumps(res, indent=1))
    print("| shape | T | hpc µs (min-max) | torch µs | torch path | speedup | bound | share of roof | TFLOP/s | GB/s |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    for r in res["rows"]:
        print(f"| {r['shape']} | {r['T']} | {r['us'][0]} ({r['us'][1]}-{r['us'][2]}) | "
              f"{r['torch_us'][0]} | {r['torch']} | {r['speedup']} | {r['bound']} | "
              f"{r['share_of_roof']} | {r['tflops']} | {r['gbs']} |")


if __name__ == "__main__":
    main()
