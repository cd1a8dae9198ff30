"""Time hpc.gemm_bf16xfp32 on the reference's route-GEMM benchmark shapes
(benchmark/route_gemm/README.md:9: N=192, K=4096, M in {2..4096}, seed 10086) next to a plain
torch fp32 matmul of the same problem (cuBLAS, the accuracy-equivalent library path). GPU box only.

    python tools/gemm_bench.py [--out route_gemm_bench.json]
"""
import argparse
import json
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO / "hpc-ops_b200"))
import torch  # noqa: E402

import hpc  # noqa: E402
from timing import card, time_graph  # noqa: E402


def _time(fn, iters, flush):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(iters):
        flush.zero_()  # 256 MB > L2: operands come from HBM every iteration
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / iters * 1e3  # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=192)
    ap.add_argument("--k", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    torch.manual_seed(10086)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ws = hpc.get_gemm_bf16xfp32_workspace(a.n, 4096)
    w = torch.randn(a.n, a.k, device="cuda", dtype=torch.float32)
    scale = 1.0 / 256
    w_high = w.to(torch.bfloat16)
    w_low = ((w - w_high.float()) / scale).to(torch.bfloat16)
    rows = []
    gpu = card()
    print(json.dumps({"card": gpu}))
    for m in [2, 4, 8, 16, 48, 96, 208, 512, 1024, 2048, 4096]:
        x = torch.randn(m, a.k, device="cuda", dtype=torch.float32).to(torch.bfloat16)
        xf = x.float()
        y = hpc.gemm_bf16xfp32(x, w_high, w_low, scale, True, True, ws)
        ref = (x.double() @ w.double().t())
        err = ((y.double() - ref).abs().max() / ref.abs().max()).item()
        assert int(ws.abs().sum().item()) == 0
        us = _time(lambda: hpc.gemm_bf16xfp32(x, w_high, w_low, scale, True, True, ws), a.iters, flush)
        us_t = _time(lambda: torch.matmul(xf, w.t()), a.iters, flush)
        f_hpc = lambda: hpc.gemm_bf16xfp32(x, w_high, w_low, scale, True, True, ws)  # noqa: E731
        f_t = lambda: torch.matmul(xf, w.t())  # noqa: E731
        try:
            gus, gus_t = time_graph(f_hpc) * 1e3, time_graph(f_t) * 1e3
        except Exception as ex:  # noqa: BLE001
            print("graph timing failed:", ex)
            gus = gus_t = float("nan")
        flops = 4.0 * m * a.n * a.k
        byts = 2.0 * m * a.k + 4.0 * a.n * a.k + 4.0 * m * a.n
        rows.append({"m": m, "split_k": hpc._ffi.lib.hpc_gemm_bf16xfp32_select_splitk(m, a.n, a.k, 1),
                     "eager_cold_us": us, "torch_fp32_eager_cold_us": us_t, "graph_us": gus,
                     "torch_fp32_graph_us": gus_t, "tflops_graph": flops / gus / 1e6,
                     "gbps_graph": byts / gus / 1e3, "rel_err_vs_fp64": err})
        print(json.dumps(rows[-1]))
    if a.out:
        Path(a.out).write_text(json.dumps({"card": gpu, "n": a.n, "k": a.k, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
