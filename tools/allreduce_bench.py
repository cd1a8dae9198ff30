"""Fused AllReduce + residual + RMSNorm benchmark (BASELINE config C5). Launch with torchrun:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node W --master-addr 127.0.0.1 \
        --master-port 29511 tools/allreduce_bench.py [--tokens 4096] [--hidden 8192]

Reports, per world size: HT path time / algbw / busbw (NCCL convention 2(W-1)/W * N / t) against
the NVLink 4 data-sheet rate (450 GB/s per direction on an H100 SXM), the LL path latency for decode-sized
batches, and NCCL all_reduce + torch RMSNorm as the unfused baseline. Max over ranks, CUDA events.
"""
import argparse
import json
import os
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "hpc-ops_b200"))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from timing import NVLINK_GBS, card, time_eager  # noqa: E402


def _rmsnorm(x, w, eps):
    """plain torch RMSNorm (fp32 math, bf16 rounding before the gamma multiply as the kernels do)"""
    xf = x.float()
    y = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)).to(torch.bfloat16)
    return (y.float() * w.float()).to(torch.bfloat16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=4096)
    ap.add_argument("--hidden", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    for k, v in (("RANK", "0"), ("WORLD_SIZE", "1"), ("LOCAL_RANK", "0"), ("MASTER_ADDR", "127.0.0.1"),
                 ("MASTER_PORT", "29533")):
        os.environ.setdefault(k, v)
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    lr = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(lr)
    dev = torch.device("cuda", lr)
    dist.init_process_group("nccl", device_id=dev)
    import hpc

    comm = hpc.MulticastCommunicator(rank, world, lr, "bench")
    T, H = a.tokens, a.hidden
    n_pad = (T + world - 1) // world * world
    g = torch.Generator(device=dev).manual_seed(10001 + rank)
    x = torch.randn((n_pad, H), generator=g, device=dev).to(torch.bfloat16)
    residual = torch.randn((n_pad, H), generator=g, device=dev).to(torch.bfloat16)
    weight = torch.randn((H,), generator=g, device=dev).to(torch.bfloat16)
    in_x, in_hdl = hpc.empty_multimem(comm, [n_pad, H], dtype=torch.bfloat16, device=dev)
    out_x, out_hdl = hpc.empty_multimem(comm, [n_pad, H], dtype=torch.bfloat16, device=dev)
    in_x.copy_(x)
    out_res = torch.empty_like(residual)
    per = n_pad // world  # rank r owns rows [r * per, (r + 1) * per)
    s, e = rank * per, (rank + 1) * per
    off = s * H * 2
    mc_in = in_hdl.get_multimem_buff((e - s, H), torch.bfloat16, off)
    mc_out = out_hdl.get_multimem_buff((e - s, H), torch.bfloat16, off)
    comm.Barrier()
    nbytes = n_pad * H * 2
    results = []
    gpu = card()
    if rank == 0:
        print(json.dumps({"card": gpu}), flush=True)

    def emit(d):
        d.update(world=world, tokens=T, hidden=H, multicast=bool(in_hdl.has_multicast))
        results.append(d)
        if rank == 0:
            print(json.dumps(d), flush=True)

    # ---- correctness spot check (rank 0 compares its slice with a NCCL reference) ----
    ref = x.float().clone()
    dist.all_reduce(ref)
    ref_res = (ref + residual.float()).to(torch.bfloat16)
    ref_out = _rmsnorm(ref_res, weight, 1e-6)

    for blocks in (32, 64, 132):
        def ht():
            hpc.fuse_allreduce_rmsnorm_high_throughput(
                in_x[s:e], mc_in, residual[s:e], weight, 1e-6, in_hdl.signal_buffer_ptrs_dev, rank,
                world, blocks, out_x[s:e], mc_out, out_res[s:e])
        ht()
        torch.cuda.synchronize()
        comm.Barrier()
        err = (out_x[s:e].float() - ref_out[s:e].float()).abs().max().item()  # own slice: residual is per rank
        ms = time_eager(ht, a.iters, warm=5, dist=dist)
        algbw = nbytes / ms / 1e6
        emit(dict(path="HT", blocks=blocks, ms=ms, algbw_gbs=algbw,
                  busbw_gbs=algbw * 2 * (world - 1) / max(world, 1), max_abs_err=err,
                  frac_nvlink_770=(algbw * 2 * (world - 1) / world / NVLINK_GBS) if world > 1 else None,
                  hbm_gbs_w1=(4 * nbytes / ms / 1e6) if world == 1 else None))

    # ---- NCCL all_reduce + torch RMSNorm (unfused baseline) ----
    buf = x.clone()

    def nccl():
        dist.all_reduce(buf)
        r = buf + residual
        _rmsnorm(r, weight, 1e-6)
    ms = time_eager(nccl, max(5, a.iters // 5), warm=5, dist=dist)
    emit(dict(path="NCCL+torch", ms=ms, algbw_gbs=nbytes / ms / 1e6))

    def nccl_only():
        dist.all_reduce(buf)
    ms = time_eager(nccl_only, max(5, a.iters // 5), warm=5, dist=dist)
    emit(dict(path="NCCL allreduce only", ms=ms, algbw_gbs=nbytes / ms / 1e6,
              busbw_gbs=nbytes / ms / 1e6 * 2 * (world - 1) / max(world, 1)))

    # ---- LL path at decode-sized batches ----
    import math
    for t_ll in (1, 8, 32, 128):
        m_pad = max(2 * math.ceil(t_ll / world) * world * 3, t_ll * world * 3)
        ws, hdl = hpc.empty_multimem(comm, [m_pad, H], dtype=torch.bfloat16, device=dev)
        ws.view(torch.int32).fill_(-2147483648)
        mc = hdl.get_multimem_buff([m_pad, H], dtype=torch.bfloat16)
        buf_bytes = (m_pad * H * 2 // 3) // 16 * 16
        flags = torch.tensor([0, 2, buf_bytes, 0, 0, 0, 0, 0, 0], dtype=torch.int32, device=dev)
        xi = x[:t_ll].contiguous()
        ri = residual[:t_ll].contiguous()
        o = torch.empty_like(xi)
        orr = torch.empty_like(ri)
        torch.cuda.synchronize()
        comm.Barrier()

        def ll():
            hpc.fuse_allreduce_rmsnorm_low_latency(xi, mc, hdl.data_buffer_ptrs_dev, ws,
                                                   flags.view(torch.uint32), world, rank, ri, weight,
                                                   1e-6, 0, o, orr, True)
        ll()
        torch.cuda.synchronize()
        err = (o.float() - ref_out[:t_ll].float()).abs().max().item()
        ms = time_eager(ll, a.iters, warm=5, dist=dist)
        emit(dict(path="LL", ll_tokens=t_ll, us=ms * 1e3, max_abs_err=err))
        xb = xi.clone()

        def nccl_small():
            dist.all_reduce(xb)
        ms2 = time_eager(nccl_small, a.iters, warm=5, dist=dist)
        emit(dict(path="NCCL allreduce only", ll_tokens=t_ll, us=ms2 * 1e3))

    if rank == 0:
        out = REPO / "gpurun_out" / f"allreduce_bench_w{world}.json"
        out.parent.mkdir(exist_ok=True)
        out.write_text(json.dumps({"card": gpu, "rows": results}, indent=1))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
