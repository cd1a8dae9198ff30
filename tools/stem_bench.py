"""Time the Stem block-mask stages and `stem_paged_kv` with CUDA events over warmed launches:

    python tools/stem_bench.py [--iters 50] [--reps 5] [--json out.json]

Each timing is the median (and min, max) of `reps` windows of `iters` launches.

Shapes: C4 (B 1, seq 32768, Hq 32, Hkv 8, page 64) and a chunked prefill (q 8192 on a 24576-token
context), both quant types. For each timing: the bytes / FLOP model from the shapes and its share
of the H100 SXM data-sheet bounds (3.35 TB/s, 989 TFLOP/s bf16 dense); the same stages written as
torch ops (the two prep stages, and GEMM + TPD, each timed under CUDA-graph replay); the C4 block-sparse prefill that consumes the mask. The
card name and power limit are read in the same run."""
import argparse
import json
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "hpc-ops_b200"))
import torch  # noqa: E402

import hpc  # noqa: E402
from timing import BF16_TFLOPS, HBM_GBS, card, spread, time_eager, time_graph  # noqa: E402

HBM = HBM_GBS * 1e9
BF16 = BF16_TFLOPS * 1e12


def inputs(q_len, kv_len, hq, hkv, quant, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    page = 64
    nblk = kv_len // page
    q = (torch.randn(q_len, hq, 128, generator=g, device="cuda") * 2).to(torch.float8_e4m3fn)
    kc = (torch.randn(nblk, page, hkv, 128, generator=g, device="cuda") * 2).to(torch.float8_e4m3fn)
    vc = torch.randn(nblk, page, hkv, 128, generator=g, device="cuda").to(torch.float8_e4m3fn)
    qscale = torch.rand(1, hq, q_len, generator=g, device="cuda") * 0.1 + 0.01
    if quant == 1:
        ks, vs = torch.ones(1, device="cuda") * 0.7, torch.ones(1, device="cuda") * 0.9
    else:
        ks = torch.rand(nblk, 2, hkv, 32, generator=g, device="cuda") + 0.5
        vs = torch.rand(hkv, generator=g, device="cuda") + 0.5
    ids = torch.randperm(nblk, generator=g, device="cuda").to(torch.int32)[None]
    cu = torch.tensor([0, q_len], dtype=torch.int32, device="cuda")
    kvl = torch.tensor([kv_len], dtype=torch.int32, device="cuda")
    return dict(q=q, kc=kc, vc=vc, qscale=qscale, ks=ks, vs=vs, ids=ids, cu=cu, kvl=kvl,
                ql=cu[1:] - cu[:-1], quant=quant)


def torch_prep(d, kv_len, q_len):
    """The two prep stages as torch ops (one request): kflat, vbias and qflat."""
    page, hkv = d["kc"].shape[1], d["kc"].shape[2]
    ids = d["ids"][0, :kv_len // page].long()
    k = d["kc"][ids].float().reshape(kv_len, hkv, 128)
    v = d["vc"][ids].float().reshape(kv_len, hkv, 128)
    if d["quant"] == 1:
        k = k * d["ks"][0]
        vs = d["vs"][0]
    else:
        k = k * d["ks"][ids].permute(0, 1, 3, 2).reshape(kv_len, hkv)[:, :, None]
        vs = d["vs"][None, :]
    kb = kv_len // 128
    kflat = k.reshape(kb, 8, 16, hkv, 128).sum(1).flip(1).permute(2, 0, 1, 3).reshape(hkv, kb, 2048)
    x = (v * vs[..., None]).norm(dim=-1).reshape(kb * 8, 16, hkv).amax(1)
    lg = torch.log(x + 1e-6)
    z = (lg - lg.mean(0)) / (lg.std(0) + 1e-6)
    vbias = (0.3 * z.clamp_min(0)).reshape(kb, 8, hkv).mean(1).T
    q = d["q"].float() * d["qscale"][0].T[:, :, None]
    qb = q_len // 128
    qflat = q.reshape(qb, 8, 16, -1, 128).sum(1).permute(2, 0, 1, 3).reshape(-1, qb, 2048)
    return kflat.bfloat16(), vbias, qflat.bfloat16()


def torch_stages(off, kflat, vbias, qflat):
    """The GEMM + TPD stages as torch ops (topk by value instead of the exact threshold)."""
    hq, hkv = qflat.shape[1], kflat.shape[1]
    k = kflat.repeat_interleave(hq // hkv, 1)
    lg = (qflat.float() @ k.float().transpose(-1, -2)) / 64 + vbias.repeat_interleave(hq // hkv, 1)[:, :, None]
    qb, kb = lg.shape[2], lg.shape[3]
    causal = torch.arange(kb, device="cuda")[None] > torch.arange(qb, device="cuda")[:, None] + off
    lg = lg.masked_fill(causal, float("-inf")).to(torch.bfloat16)
    kk = min(kb, 60)
    top = lg.topk(kk, -1).indices
    return torch.zeros_like(lg, dtype=torch.uint8).scatter_(-1, top, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    res = {"card": card(), "rows": []}
    print(json.dumps({"card": res["card"]}))

    def us(timer):  # median, min, max in µs of a.reps windows
        return [t * 1e3 for t in spread(timer, a.reps)]

    for name, q_len, kv_len in (("C4", 32768, 32768), ("chunked", 8192, 24576)):
        for quant in (1, 0):
            d = inputs(q_len, kv_len, 32, 8, quant)
            qt = hpc.QuantType(quant)
            hq, hkv = 32, 8
            qb, kb = (q_len + 127) // 128, (kv_len + 127) // 128
            prep_kv = lambda: hpc.stem_oam_prep_paged_kv(d["kc"], d["vc"], d["ks"], d["vs"], d["ids"],
                                                         d["kvl"], 0.3, quant_type=qt)
            prep_q = lambda: hpc.stem_oam_prep_varlen_q(d["q"], d["qscale"], d["ql"], d["cu"])
            kflat, vbias = prep_kv()
            qflat = prep_q()
            gemm = lambda: hpc.stem_oam_gemm(qflat, kflat, vbias, d["ql"], d["kvl"])
            lg = gemm()
            tpd = lambda: hpc.stem_tpd(lg, d["ql"], d["kvl"], d["kvl"])
            full = lambda: hpc.stem_paged_kv(d["q"], d["kc"], d["vc"], d["qscale"], d["ks"], d["vs"],
                                             d["ids"], d["cu"], d["kvl"], d["kvl"], quant_type=qt)
            mask = full()
            kv_bytes = 2 * kv_len * hkv * 128
            flat_kv = hkv * kb * 2048 * 2
            flat_q = hq * qb * 2048 * 2
            logit_b = hq * qb * kb * 2
            mask_b = hq * qb * kb
            causal_frac = min(1.0, (kb - qb + (qb + 1) / 2) / kb)
            gemm_flop = 2 * hq * qb * kb * 2048 * causal_frac
            model = {
                "prep_kv": (kv_bytes + flat_kv, 0), "prep_q": (q_len * hq * 128 + flat_q, 0),
                "gemm": (flat_kv + flat_q + logit_b, gemm_flop), "tpd": (logit_b + mask_b, 0),
                "stem_paged_kv": (kv_bytes + q_len * hq * 128 + 2 * (flat_kv + flat_q) + 2 * logit_b + mask_b,
                                  gemm_flop),
            }
            # the same stages as torch ops, replayed from CUDA graphs
            off = (kv_len - q_len + 127) // 128
            t_torch = us(lambda: time_graph(lambda: torch_stages(off, kflat, vbias, qflat), 1, a.iters))
            t_torch_prep = us(lambda: time_graph(lambda: torch_prep(d, kv_len, q_len), 1, a.iters))
            prefill = lambda: hpc.attention_with_kvcache_blocksparse_prefill_fp8(
                d["q"], d["kc"], d["vc"], d["qscale"], d["ks"], d["vs"], d["cu"], d["ids"], d["kvl"],
                q_len, qt, block_mask=mask)
            t_prefill = time_eager(prefill, max(5, a.iters // 5)) * 1e3
            for stage, fn in (("prep_kv", prep_kv), ("prep_q", prep_q), ("gemm", gemm), ("tpd", tpd),
                              ("stem_paged_kv", full)):
                t, lo, hi = us(lambda: time_eager(fn, a.iters))
                by, fl = model[stage]
                floor = max(by / HBM, fl / BF16) * 1e6
                row = dict(shape=name, quant=quant, stage=stage, us=round(t, 2), us_min=round(lo, 2),
                           us_max=round(hi, 2), bytes=by, flop=fl, floor_us=round(floor, 2),
                           share=round(floor / t, 3), bound="hbm" if by / HBM >= fl / BF16 else "bf16")
                if stage == "gemm":
                    row["torch_gemm_tpd_us"] = [round(x, 1) for x in t_torch]
                if stage == "prep_kv":
                    row["torch_prep_kv_q_us"] = [round(x, 1) for x in t_torch_prep]
                if stage == "stem_paged_kv":
                    row["prefill_with_mask_us"] = round(t_prefill, 1)
                    row["density"] = round(float(mask.float().mean()), 4)
                print(json.dumps(row))
                res["rows"].append(row)
    if a.json:
        Path(a.json).parent.mkdir(parents=True, exist_ok=True)
        Path(a.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
