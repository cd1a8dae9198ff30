"""Time fused RMSNorm -> FP8 and the masked per-expert activation quantisers against the same
computation written as torch ops:

    python tools/norm_act_bench.py [--iters 50] [--reps 5] [--json out.json]

Every figure is kernel time from CUDA events around `iters` replays of a CUDA graph holding one
call, the median (and min, max) of `reps` warmed windows. The torch version is captured and timed
the same way. For each shape: the algorithmic bytes (RMSNorm: x, weight and outputs; masked ops:
valid rows only) and their share of the H100 SXM data-sheet 3.35 TB/s. The card's name, power limit
and max SM clock are read in the same run.

Shapes: RMSNorm at T in {1, 16, 128, 1024, 8192, 32768} x H in {4096, 5120, 7168} x is_moe, plus
H = 1024 (one warp per row; 4096 takes four and 5120 / 7168 eight); masked ops at E 32, T_max 1024,
C 2048 with 100 %, 50 % and 10 % of the rows valid, per-tensor and blockwise."""
import argparse
import json
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "hpc-ops_b200"))
import torch  # noqa: E402

import hpc  # noqa: E402
from timing import HBM_GBS, card, spread, time_graph  # noqa: E402

HBM = HBM_GBS * 1e9


def graphed_us(fn, a):
    """Median, min and max in µs of `a.reps` windows of `a.iters` replays of a graph of one call."""
    return [t * 1e3 for t in spread(lambda: time_graph(fn, 1, a.iters), a.reps)]


def torch_rmsnorm(x, w, sc, eps, is_moe):
    y = x.float() * w.float() * torch.rsqrt(x.float().pow(2).mean(-1, keepdim=True) + eps)
    q0 = (y / sc[0]).clamp(-448, 448).to(torch.float8_e4m3fn)
    if is_moe:
        return y, q0, (y / sc[1]).clamp(-448, 448).to(torch.float8_e4m3fn)
    return q0


def torch_masked(gu, cnt, T, sc, blockwise):
    """All rows (the torch chain has no cheap way to skip them), invalid rows restored after."""
    g, u = gu.float().chunk(2, -1)
    v = g / (1 + torch.exp(-g)) * u
    keep = (torch.arange(T, device=gu.device)[None] < cnt[:, None]).reshape(-1, 1)
    if blockwise:
        amax = v.abs().reshape(v.shape[0], -1, 128).amax(-1)
        s = amax / 448
        q = (v * (1 / (s + 1e-8)).repeat_interleave(128, -1)).to(torch.float8_e4m3fn)
        return torch.where(keep, q.view(torch.uint8), 0), torch.where(keep, s, 0)
    q = (v * sc[0]).clamp(-448, 448).to(torch.float8_e4m3fn)
    return torch.where(keep, q.view(torch.uint8), 0)


def row(name, by, t_ours, t_torch, **kw):
    t, lo, hi = t_ours
    r = dict(op=name, **kw, us=round(t, 2), us_min=round(lo, 2), us_max=round(hi, 2), bytes=by,
             hbm_share=round(by / HBM * 1e6 / t, 3), torch_us=[round(v, 2) for v in t_torch],
             speedup=round(t_torch[0] / t, 2))
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    res = {"card": card(), "rows": []}
    print(json.dumps({"card": res["card"]}), flush=True)
    eps = 1e-6
    sc = torch.tensor([0.05, 0.5], device="cuda")
    shapes = [(T, H) for H in (4096, 5120, 7168) for T in (1, 16, 128, 1024, 8192, 32768)]
    shapes += [(T, 1024) for T in (1, 1024, 32768)]
    for T, H in shapes:
        x = torch.randn(T, H, device="cuda").to(torch.bfloat16)
        w = torch.rand(H, device="cuda").to(torch.bfloat16)
        for moe in (False, True):
            ours = lambda: hpc.fused_rmsnorm_with_scale(x, w, eps, sc, moe)  # noqa: E731
            ref = lambda: torch_rmsnorm(x, w, sc, eps, moe)  # noqa: E731
            by = T * H * 2 + H * 2 + T * H * (6 if moe else 1)
            res["rows"].append(row("rmsnorm", by, graphed_us(ours, a), graphed_us(ref, a),
                                   T=T, H=H, is_moe=moe))
        del x
    E, T, C = 32, 1024, 2048
    gu = torch.randn(E * T, 2 * C, device="cuda").to(torch.bfloat16)
    out = torch.empty(E * T, C, dtype=torch.float8_e4m3fn, device="cuda")
    osc = torch.empty(E * T, C // 128, device="cuda")
    for fill in (1.0, 0.5, 0.1):
        cnt = torch.full((E,), int(T * fill), dtype=torch.int32, device="cuda")
        valid = E * int(T * fill)
        for blockwise in (False, True):
            if blockwise:
                ours = lambda: hpc.masked_act_mul_and_blockwise_quant(gu, cnt, out, osc)  # noqa: E731
            else:
                ours = lambda: hpc.masked_act_mul_and_quant(gu, sc[:1], cnt, out)  # noqa: E731
            ref = lambda: torch_masked(gu, cnt, T, sc, blockwise)  # noqa: E731
            by = valid * (4 * C + C + (4 * C // 128 if blockwise else 0))
            res["rows"].append(row("masked_blockwise" if blockwise else "masked_pertensor", by,
                                   graphed_us(ours, a), graphed_us(ref, a),
                                   E=E, T_max=T, C=C, fill=fill))
    if a.json:
        Path(a.json).parent.mkdir(parents=True, exist_ok=True)
        Path(a.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
