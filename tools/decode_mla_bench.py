"""Time hpc.attention_decode_mla_bf16 (absorbed MLA decode, DeepSeek-V3 latent head 576 / 512) on
the GPU box, attention + combine with a pre-assigned task map, pages in random order.

    python tools/decode_mla_bench.py [--heads 16,128] [--batch 1,32,128] [--ctx 2048,8192,32768]
                                     [--mtp 0,1] [--probe]

Per shape: eager launches and graph replay (median and spread of repeated windows), the
algorithmic bytes (sum n_b * 1152 for the cache, counted once whatever the number of query tiles,
plus Q and the output), the achieved GB/s and its fraction of the data-sheet HBM bandwidth, and
the speedup over a torch chain (page gather -> bf16 matmul -> softmax -> matmul) where that chain
fits in memory. --probe rebuilds the kernel a second time as a producer-only build (consumers wait
for the pages and do no math) and a consumer-only build (no loads), into a temporary directory,
and times them on the same shapes: what bounds the kernel is read off those two.
One JSON line per shape, and the card first.
"""
import argparse
import ctypes
import json
import math
import shutil
import subprocess
import sys
import tempfile
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "hpc-ops_b200"))
sys.path.insert(0, str(REPO / "tools"))
import torch  # noqa: E402

import hpc  # noqa: E402
from timing import card, peaks, spread, time_eager, time_graph  # noqa: E402

SCALE = (0.1 * math.log(40.0) + 1.0) ** 2 / math.sqrt(192.0)


def _probe_lib(mode, tmp):
    """_C.so rebuilt with HPC_DECODE_MLA_PROBE=mode (1: no math, 2: no loads)."""
    sys.path.insert(0, str(REPO / "hpc-ops_b200"))
    import build as b
    csrc = REPO / "hpc-ops_b200" / "csrc"
    objs = []
    for src in sorted(csrc.glob("*.cu")):
        if src.stem in ("decode_attn_mla", "host_utils", "version"):
            obj = Path(tmp) / f"{src.stem}_{mode}.o"
            extra = [f"-DHPC_DECODE_MLA_PROBE={mode}"] if src.stem == "decode_attn_mla" else []
            if src.stem == "version":
                extra = ["-include", str(REPO / "hpc-ops_b200" / "build" / "obj" / "built_info.h")]
            subprocess.run([b._nvcc(), *b.NVCC_FLAGS, *extra, "-c", str(src), "-o", str(obj)],
                           check=True, capture_output=True)
            objs.append(str(obj))
    so = Path(tmp) / f"probe_{mode}.so"
    subprocess.run([b._nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", *objs,
                    "-lcuda", "-o", str(so)], check=True, capture_output=True)
    lib = ctypes.CDLL(str(so))
    ref = hpc._ffi.lib.hpc_attention_decode_mla_bf16_async
    fn = lib.hpc_attention_decode_mla_bf16_async
    fn.restype, fn.argtypes = ref.restype, ref.argtypes
    return fn


def _inputs(B, H, mtp, ctx, g):
    sq = mtp + 1
    npg = (ctx + 63) // 64
    nblk = B * npg
    kv = torch.randn(nblk, 64, 576, device="cuda", dtype=torch.bfloat16)
    q = (torch.randn(B * sq, H, 576, device="cuda") * 0.05).to(torch.bfloat16)
    ids = torch.randperm(nblk, device="cuda", generator=g).to(torch.int32).reshape(B, npg)
    lens = torch.full((B,), ctx, dtype=torch.int32, device="cuda")
    return q, kv, ids, lens


def _torch_chain(q, kv, ids, lens, mtp):
    B, npg = ids.shape
    sq = mtp + 1
    H = q.size(1)
    n = int(lens[0])
    k = kv[ids.long()].reshape(B, npg * 64, 576)[:, :n]
    qb = q.reshape(B, sq * H, 576)
    s = torch.matmul(qb, k.transpose(1, 2)).float() * SCALE
    j = torch.arange(n, device=q.device)
    lim = n - sq + torch.arange(sq, device=q.device).repeat_interleave(H)
    s.masked_fill_(j[None, None, :] > lim[None, :, None], float("-inf"))
    p = torch.softmax(s, -1).to(torch.bfloat16)
    return torch.matmul(p, k[..., :512]).reshape(B * sq, H, 512)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--heads", default="16,128")
    ap.add_argument("--batch", default="1,32,128")
    ap.add_argument("--ctx", default="2048,8192,32768")
    ap.add_argument("--mtp", default="0,1")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--probe", action="store_true")
    a = ap.parse_args()
    pk = peaks()
    print(json.dumps({"card": card(), "hbm_gbs_datasheet": pk["hbm_gbs"], "peaks_source": pk["source"]}))
    tmp = tempfile.mkdtemp(prefix="mla_probe_")
    probes = {}
    if a.probe:
        for mode in (1, 2):
            probes[mode] = _probe_lib(mode, tmp)
    g = torch.Generator(device="cuda").manual_seed(0)
    ctas = hpc._ffi.sm_count()
    try:
        for H in map(int, a.heads.split(",")):
            for mtp in map(int, a.mtp.split(",")):
                for B in map(int, a.batch.split(",")):
                    for ctx in map(int, a.ctx.split(",")):
                        sq = mtp + 1
                        q, kv, ids, lens = _inputs(B, H, mtp, ctx, g)
                        T = hpc.mla_num_query_tiles(H, mtp)
                        tm = hpc.get_attention_decode_task_workspace(B, ids.size(1) * 64 + sq, T,
                                                                     512)
                        hpc.assign_attention_decode_task(lens, tm, T, sq, True, 512)
                        y = torch.empty(B * sq, H, 512, dtype=torch.bfloat16, device="cuda")

                        def run():
                            hpc.attention_decode_mla_bf16(q, kv, ids, lens, SCALE, mtp=mtp,
                                                          new_kv_included=True, task_map=tm,
                                                          output=y)
                        eager = spread(lambda: time_eager(run, 20), a.reps)
                        graph = spread(lambda: time_graph(run, reps=10, iters=5), a.reps)
                        nbytes = B * ctx * 1152 + q.numel() * 2 + y.numel() * 2
                        gbs = nbytes / (graph[0] * 1e-3) / 1e9
                        rec = dict(H=H, B=B, ctx=ctx, mtp=mtp, T=T, bytes=nbytes,
                                   eager_ms=eager, graph_ms=graph, graph_gbs=round(gbs, 1),
                                   frac_datasheet_hbm=round(gbs / pk["hbm_gbs"], 3))
                        chain_bytes = B * ctx * (1152 * 2 + sq * H * 6)
                        if chain_bytes < 30e9:
                            tc = spread(lambda: time_eager(lambda: _torch_chain(q, kv, ids, lens,
                                                                                mtp), 3), 3)
                            rec["torch_chain_ms"] = tc
                            rec["speedup_vs_torch"] = round(tc[0] / graph[0], 2)
                        if probes:
                            ws = torch.empty(2 * ctas * 64 * 513 + ctas * (256 * 128 + 512),
                                             dtype=torch.float32, device="cuda")
                            # zeroed: the producer-only build writes no chunk_base, which the
                            # combine still reads (slot 2c of bin 0 is in range for every c)
                            cb = torch.zeros(B * T, dtype=torch.int32, device="cuda")
                            for mode, fn in probes.items():
                                def prun(fn=fn):
                                    fn(y.data_ptr(), ws.data_ptr(), cb.data_ptr(), tm.data_ptr(),
                                       q.data_ptr(), kv.data_ptr(), ids.data_ptr(), B, sq, H, 576,
                                       kv.size(0), 64, ids.size(1), y.stride(0), q.stride(0),
                                       kv.stride(0), kv.stride(1), SCALE, ctas,
                                       torch.cuda.current_stream().cuda_stream)
                                name = "producer_only_ms" if mode == 1 else "consumer_only_ms"
                                rec[name] = spread(lambda: time_eager(prun, 20), a.reps)
                        print(json.dumps(rec), flush=True)
                        del q, kv, ids, lens, tm, y
                        torch.cuda.empty_cache()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
