"""Does the DRAM access granule limit decode? Times fp8 and bf16 paged decode at the C2 shape with the
cache in NHD (a head's token rows are 128 B / 256 B runs strided by Hkv rows) and in HND (a head's
page is one contiguous 8 KB / 16 KB run). GPU box only.

    python tools/decode_layout_probe.py
"""
import json
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "hpc-ops_b200"))
import torch  # noqa: E402

import hpc  # noqa: E402
from timing import card, peaks, time_eager  # noqa: E402


def main():
    dev = "cuda"
    B, ctx, hq, hkv, D, bs = 64, 8192, 32, 8, 128, 64
    nb = ctx // bs
    pk = peaks()
    out = {"card": card()}
    g = torch.Generator(device=dev).manual_seed(0)
    ids = torch.randperm(B * nb, device=dev).to(torch.int32).view(B, nb)
    lens = torch.full((B,), ctx, dtype=torch.int32, device=dev)
    tm = hpc.get_attention_decode_task_workspace(B, ctx, hkv, 64)
    hpc.assign_attention_decode_task(lens, tm, hkv, 1, True, 64)
    for dtype, name, eb in ((torch.float8_e4m3fn, "fp8", 1), (torch.bfloat16, "bf16", 2)):
        for layout in ("NHD", "HND"):
            kv = torch.randn(B * nb, 2, bs, hkv, D, device=dev, generator=g).to(dtype)
            if layout == "HND":
                kv = kv.permute(0, 1, 3, 2, 4).contiguous().permute(0, 1, 3, 2, 4)
            q = torch.randn(B, hq, D, device=dev, generator=g).to(dtype)
            y = torch.empty(B, hq, D, device=dev, dtype=torch.bfloat16)
            if eb == 1:
                qs = torch.ones(B, hq, device=dev)
                one = torch.ones(1, device=dev)
                fn = lambda: hpc.attention_decode_fp8(q, kv[:, 0], kv[:, 1], ids, lens, qs, one, one,  # noqa: E731
                                                      new_kv_included=True, task_map=tm, output=y)
            else:
                fn = lambda: hpc.attention_decode_bf16(q, kv[:, 0], kv[:, 1], ids, lens,  # noqa: E731
                                                       new_kv_included=True, task_map=tm, output=y)
            ms = time_eager(fn, 50)
            byts = 2 * B * ctx * hkv * D * eb
            out[f"{name}_{layout}"] = {"ms": round(ms, 5), "gbs": round(byts / ms / 1e6, 1),
                                       "frac_hbm": round(byts / ms / 1e6 / pk["hbm_gbs"], 4)}
            del kv
    print(json.dumps(out))


if __name__ == "__main__":
    main()
