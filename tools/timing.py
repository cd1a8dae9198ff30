"""How the benchmarks time, written once: CUDA-event timers over eager launches and over CUDA-graph
replays, the spread of repeated windows, the H100 SXM data-sheet peaks and a read of the card the
figures come from. Imported by bench_extras.py and by the per-op tools, which only describe their
workloads."""
import json
import subprocess
from pathlib import Path

import torch

REPO = Path(__file__).resolve().parents[1]

# H100 SXM data sheet, dense rates, for a card allowed 700 W (not measured)
HBM_GBS = 3350.0      # HBM3
BF16_TFLOPS = 989.0
FP8_TFLOPS = 1979.0   # e4m3
NVLINK_GBS = 450.0    # NVLink 4, per direction


def peaks():
    f = REPO / "MEASURED_PEAKS.json"
    d = {"hbm_gbs": HBM_GBS, "bf16_tflops": BF16_TFLOPS, "source": "H100 SXM data sheet (not measured)"}
    if f.exists():
        try:
            j = json.loads(f.read_text())
            d = {"hbm_gbs": float(j["hbm_gbs"]), "bf16_tflops": float(j["bf16_tflops"]),
                 "source": "measured (MEASURED_PEAKS.json)"}
        except Exception:
            pass
    # no measured FP8 entry exists: 2x the measured cuBLAS bf16 burst is the practical tensor roof
    d["fp8_tflops_2x_bf16"] = 2 * d["bf16_tflops"]
    return d


def _max_over_ranks(ms, dist):
    t = torch.tensor([ms], dtype=torch.float64, device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def time_eager(fn, iters, warm=3, dist=None):
    """ms per call: `iters` back-to-back eager calls after `warm` untimed ones.
    With `dist` the ranks start together and the maximum over ranks is returned."""
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    if dist is not None:
        dist.barrier()
        torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    return ms if dist is None else _max_over_ranks(ms, dist)


def time_graph(fn, reps=20, iters=5, dist=None):
    """ms per call: `reps` back-to-back calls captured in one CUDA graph, replayed `iters` times
    (the reference harness times graph replays: benchmark/fuse_allreduce_rmsorm/...:116-170).
    With `dist` the ranks start together and the maximum over ranks is returned."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    if dist is not None:
        dist.barrier()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    torch.cuda.synchronize()
    if dist is not None:
        dist.barrier()
        torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / (iters * reps)
    if dist is not None:
        ms = _max_over_ranks(ms, dist)
    del g
    return ms


def spread(timer, reps):
    """(median, min, max) of `reps` calls of `timer`, a zero-argument callable that returns ms."""
    t = sorted(timer() for _ in range(reps))
    return t[len(t) // 2], t[0], t[-1]


def card():
    """Name, power limit, max and current SM clock of the first GPU, read in the run whose figures
    they qualify (a power-limited card runs below the data-sheet rates)."""
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                          "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    name, power, max_sm, sm = [s.strip() for s in out.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": max_sm, "sm_clock": sm}
