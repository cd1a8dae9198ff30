"""Time hpc.gemm_blockwise_fp8 on DeepSeek-V3 and Qwen3 projection shapes next to three baselines on
the same operands: torch bf16 matmul on the dequantised weight, hpc.group_gemm_blockwise_fp8 with
one group (scales re-laid out outside the timed region) and torch._scaled_mm with 1x128 x 128x128
block scales where this torch / cuBLAS accepts it. Every time is a CUDA-graph replay
(tools/timing.py); the card's name, power limit and SM clock are read in the same run.
GPU box only.

    python tools/gemm_fp8_bench.py [--ms 1,64,4096] [--out gemm_fp8_bench.json]

Per row: time (us), TFLOP/s (2MNK), bytes (MK + NK + 2MN plus both scale tensors), the share of the
roof (least time = max(FLOP / 1979 TFLOP/s, bytes / 3.35 TB/s), data-sheet figures, over the kernel
time, with the bound that sets it) and the K split hpc_gemm_blockwise_fp8_config chose.
"""
import argparse
import json
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO / "hpc-ops_b200"))
sys.path.insert(0, str(REPO))
import torch  # noqa: E402

import hpc  # noqa: E402
from oracle.moe_exact import scale_granule  # noqa: E402
from synth.gemm_blockwise import dequant_weight  # noqa: E402
from timing import FP8_TFLOPS, HBM_GBS, card, time_graph  # noqa: E402

SHAPES = [("dsv3_q_a_kv_a", 2112, 7168), ("dsv3_q_b", 24576, 1536), ("dsv3_kv_b", 32768, 512),
          ("dsv3_o", 7168, 16384), ("dsv3_shared_gate_up", 4096, 7168),
          ("dsv3_shared_down", 7168, 2048), ("qwen3_32b_gate_up", 10240, 5120),
          ("qwen3_32b_o", 5120, 8192), ("qwen3_32b_down", 5120, 25600),
          ("qwen3_8b_qkv", 6144, 4096), ("qwen3_8b_gate_up", 24576, 4096)]


def _operands(m, n, k, g):
    a = torch.randn((m, k), generator=g, device="cuda").to(torch.bfloat16)
    x, xs = hpc.blockwise_fp8_quant(a)
    nb, kb = (n + 127) // 128, k // 128
    wf = torch.randn((nb * 128, k), generator=g, device="cuda") * 0.02
    blk = wf.view(nb, 128, kb, 128)
    ws = (blk.abs().amax((1, 3)) / 448.0).float().contiguous()
    w = (blk / ws[:, None, :, None]).clamp(-448, 448).view(nb * 128, k)[:n].to(torch.float8_e4m3fn)
    return x, xs, w.contiguous(), ws


def _try(make):
    try:
        fn = make()
        fn()
        torch.cuda.synchronize()
        return time_graph(fn, reps=10, iters=10) * 1e3, None
    except Exception as e:  # a baseline this build or library does not support
        torch.cuda.synchronize()
        return None, f"{type(e).__name__}: {str(e).splitlines()[0][:120]}"


def _grouped(x, xs, w, ws, m, n, k):
    seq = torch.tensor([m], dtype=torch.int32, device="cuda")
    cu = torch.tensor([0, m], dtype=torch.int32, device="cuda")
    kb = k // 128
    gran = scale_granule(m)
    xs_pad = torch.zeros(((m + gran - 1) // gran * gran, kb), device="cuda")
    xs_pad[:m] = xs
    ws4 = torch.zeros((1, ws.size(0), (kb + 3) // 4 * 4), device="cuda")
    ws4[0, :, :kb] = ws
    xst = hpc.reformat_x_scale(xs_pad, seq, cu, m)
    w3 = w.unsqueeze(0)
    return lambda: hpc.group_gemm_blockwise_fp8(x, w3, seq, cu, xst, ws4, m)


def _scaled_mm(x, xs, w, ws):
    from torch.nn.functional import ScalingType, SwizzleType, scaled_mm

    return lambda: scaled_mm(x, w.t(), xs, ScalingType.BlockWise1x128, ws,
                             ScalingType.BlockWise128x128, swizzle_a=SwizzleType.NO_SWIZZLE,
                             swizzle_b=SwizzleType.NO_SWIZZLE, output_dtype=torch.bfloat16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ms", default="1,8,64,256,1024,4096")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    for name, n, k in SHAPES:
        for m in (int(s) for s in a.ms.split(",")):
            x, xs, w, ws = _operands(m, n, k, g)
            wd = dequant_weight(w, ws).to(torch.bfloat16)
            ad = (x.float() * xs.repeat_interleave(128, 1)).to(torch.bfloat16)
            t_new, err = _try(lambda: lambda: hpc.gemm_blockwise_fp8(x, xs, w, ws))
            assert err is None, err
            t_bf16, _ = _try(lambda: lambda: ad @ wd.t())
            t_grp, grp_err = _try(lambda: _grouped(x, xs, w, ws, m, n, k))
            t_smm, smm_err = _try(lambda: _scaled_mm(x, xs, w, ws))
            flop = 2.0 * m * n * k
            byts = m * k + n * k + 2 * m * n + 4 * (xs.numel() + ws.numel())
            t_flop, t_byte = flop / (FP8_TFLOPS * 1e12) * 1e6, byts / (HBM_GBS * 1e9) * 1e6
            r = dict(shape=name, m=m, n=n, k=k,
                     split=hpc._ffi.lib.hpc_gemm_blockwise_fp8_config(m, n, k),
                     us=round(t_new, 2), tflops=round(flop / t_new / 1e6, 1), bytes=byts,
                     roof_share=round(max(t_flop, t_byte) / t_new, 3),
                     bound="fp8" if t_flop >= t_byte else "hbm",
                     bf16_matmul_us=round(t_bf16, 2),
                     grouped_us=round(t_grp, 2) if t_grp else grp_err,
                     scaled_mm_us=round(t_smm, 2) if t_smm else f"unsupported ({smm_err})")
            rows.append(r)
            print(json.dumps(r), flush=True)
            del x, xs, w, ws, wd, ad
    res = dict(card=card(), rows=rows)
    print(json.dumps(res["card"]))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
