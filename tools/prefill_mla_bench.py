"""Kernel time of hpc.attention_prefill_mla_bf16 against two torch SDPA baselines, alternated
round by round in one run (CUDA events, tools/timing.py):

  flash     SDPBackend.FLASH_ATTENTION on the usual workaround: k_pe expanded to every head and
            concatenated to k_nope, V zero-padded from 128 to 192 (its extra 64 output columns
            dropped)
  efficient SDPBackend.EFFICIENT_ATTENTION on the same K, V unpadded (128)

Only the attention call is timed for the baselines: the expansion and padding they need are left
out, which favours them. Self-attention shapes use is_causal; chunked prefill (new tokens over a
prefix) uses causal_lower_right. A backend that refuses a shape is reported as unavailable.
All shapes use the DeepSeek-V3 softmax scale. FLOP = 2 (192 + 128) H x visible (query, key)
pairs; the share is of the 989 TFLOP/s data-sheet bf16 rate.

    python tools/prefill_mla_bench.py [--heads 16,128] [--seq 4096,8192,16384,32768] [--reps 5]
"""
import argparse
import json
import math
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "hpc-ops_b200"))
sys.path.insert(0, str(REPO / "tools"))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
from torch.nn.attention import SDPBackend, sdpa_kernel  # noqa: E402
from torch.nn.attention.bias import causal_lower_right  # noqa: E402

import hpc  # noqa: E402
from timing import BF16_TFLOPS, card, spread, time_eager  # noqa: E402

SCALE = (0.1 * math.log(40.0) + 1.0) ** 2 / math.sqrt(192.0)


def visible_pairs(nq, nk):
    return sum(max(0, min(nk, nk - nq + i + 1)) for i in range(nq))


def _shape(H, nb, nq, nk, g):
    """nb requests of nq new tokens over nk keys each (nk - nq of them a prefix)."""
    tq, tkv = nb * nq, nb * nk
    q = torch.randn(tq, H, 192, generator=g, device="cuda").to(torch.bfloat16)
    kv = torch.randn(tkv, H, 256, generator=g, device="cuda").to(torch.bfloat16)
    latent = torch.randn(tkv, 576, generator=g, device="cuda").to(torch.bfloat16)
    cu_q = torch.arange(nb + 1, dtype=torch.int32, device="cuda") * nq
    cu_kv = torch.arange(nb + 1, dtype=torch.int32, device="cuda") * nk
    return q, kv, latent, cu_q, cu_kv


def _sdpa_inputs(q, kv, latent, H, nb, nq, nk):
    """[nb, H, S, D] tensors of the workaround: k = [k_nope | k_pe expanded], v padded or not."""
    qb = q.view(nb, nq, H, 192).transpose(1, 2)
    kn = kv[..., :128].reshape(nb, nk, H, 128)
    kp = latent[:, 512:].reshape(nb, nk, 1, 64).expand(nb, nk, H, 64)
    kb = torch.cat([kn, kp], 3).transpose(1, 2).contiguous()
    vb = kv[..., 128:].reshape(nb, nk, H, 128).transpose(1, 2).contiguous()
    vpad = F.pad(vb, (0, 64))
    return qb.contiguous(), kb, vb, vpad


def _sdpa(backend, qb, kb, vb, nq, nk):
    mask = None if nq == nk else causal_lower_right(nq, nk)
    with sdpa_kernel([backend]):
        if mask is None:
            return F.scaled_dot_product_attention(qb, kb, vb, is_causal=True, scale=SCALE)
        return F.scaled_dot_product_attention(qb, kb, vb, attn_mask=mask, scale=SCALE)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--heads", default="16,128")
    ap.add_argument("--seq", default="4096,8192,16384,32768")
    ap.add_argument("--chunked", default="4x2048+16384", help="requests x new tokens + prefix")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    print(json.dumps({"card": card(), "bf16_tflops_datasheet": BF16_TFLOPS}), flush=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    shapes = [(1, s, s) for s in map(int, a.seq.split(","))]
    if a.chunked:
        nb, rest = a.chunked.split("x")
        new, prefix = map(int, rest.split("+"))
        shapes.append((int(nb), new, new + prefix))
    for H in map(int, a.heads.split(",")):
        for nb, nq, nk in shapes:
            q, kv, latent, cu_q, cu_kv = _shape(H, nb, nq, nk, g)
            y = torch.empty(nb * nq, H, 128, dtype=torch.bfloat16, device="cuda")

            def ours():
                hpc.attention_prefill_mla_bf16(q, kv[..., :128], latent[:, 512:], kv[..., 128:],
                                               cu_q, cu_kv, nq, SCALE, output=y)

            qb, kb, vb, vpad = _sdpa_inputs(q, kv, latent, H, nb, nq, nk)
            base = {"flash": (SDPBackend.FLASH_ATTENTION, vpad),
                    "efficient": (SDPBackend.EFFICIENT_ATTENTION, vb)}
            runs = {"ours": ours}
            rec = dict(H=H, requests=nb, new_tokens=nq, keys=nk)
            ours()
            torch.cuda.synchronize()
            mine = y.view(nb, nq, H, 128).transpose(1, 2).float()
            for name, (be, vv) in base.items():
                try:
                    out = _sdpa(be, qb, kb, vv, nq, nk)
                    torch.cuda.synchronize()
                except RuntimeError as e:
                    rec[f"{name}_ms"] = f"unavailable: {str(e).splitlines()[0][:120]}"
                    continue
                rec[f"max_abs_diff_{name}"] = float((out[..., :128].float() - mine).abs().max())
                del out
                runs[name] = (lambda be=be, vv=vv: _sdpa(be, qb, kb, vv, nq, nk))
            times = {k: [] for k in runs}
            for _ in range(a.reps):  # alternate the contenders round by round
                for k, fn in runs.items():
                    times[k].append(spread(lambda fn=fn: time_eager(fn, a.iters), 1)[0])
            flop = 2 * (192 + 128) * H * nb * visible_pairs(nq, nk)
            for k, t in times.items():
                t = sorted(t)
                med = t[len(t) // 2]
                rec[f"{k}_ms"] = [round(med, 4), round(t[0], 4), round(t[-1], 4)]
                rec[f"{k}_tflops"] = round(flop / (med * 1e-3) / 1e12, 1)
                rec[f"{k}_frac_datasheet"] = round(flop / (med * 1e-3) / 1e12 / BF16_TFLOPS, 3)
            for name in base:
                if name in times:
                    rec[f"speedup_vs_{name}"] = round(rec[f"{name}_ms"][0] / rec["ours_ms"][0], 2)
            print(json.dumps(rec), flush=True)
            del q, kv, latent, qb, kb, vb, vpad, y, mine
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
