"""Seeded inputs for the MLA prefill (csrc/prefill_mla.cu, oracle/prefill_mla.py).

A case is a dict: q [Tq, H, 192] bf16; k_nope / v [Tkv + SLACK, H, 128], the two halves of one
[Tkv + SLACK, H, 256] buffer (a kv_b_proj output); k_pe [Tkv + SLACK, 64], columns 512.. of a
[Tkv + SLACK, 576] latent buffer whose other columns hold NaN; cu_seqlens_q / cu_seqlens_kv
[B + 1] int32; max_q; scale; and the buffers themselves ("kv", "latent"). The SLACK rows past the
last request's keys hold NaN in K, k_pe and V: a kernel that lets a key past a request's last one
into a row (through its score or through 0 * v) writes NaN there.

Kinds (scores spread to |s| ~ 50 in all of them):
  random  q, k_nope, k_pe, v ~ N(0, 1)-shaped: every key, head and tile carries weight
  pe      q_nope = 0: q_nope . k_nope is 0 and the scores come from the 64 k_pe columns alone
  edge    position codes in k_nope over the buffer row index g: key g is (cos t_f g, sin t_f g)
          over 64 random frequencies t_f, and query i of a request points at g = kv0 + nk - nq + i
          + 1/2, so its highest-scoring keys are the one at its causal edge and the one past it.
          The first key of every request after the first has V = POISON_V: it is the key one past
          the previous request's last row.
"""
import math

import torch

from oracle.prefill_mla import D_NOPE, D_PE, DQK, DV

KINDS = ("random", "pe", "edge")
SLACK = 5
POISON_V = 1000.0
EDGE_A = 24.0
SCALE_DSV3 = (0.1 * math.log(40.0) + 1.0) ** 2 / math.sqrt(192.0)  # mscale^2 / sqrt(qk_head_dim)


def _cu(lens):
    return torch.tensor([0] + list(lens), dtype=torch.int64).cumsum(0).to(torch.int32)


def _codes(g, freqs):
    ang = g.double()[:, None] * freqs[None, :]
    return torch.stack([ang.cos(), ang.sin()], -1).reshape(-1, 2 * freqs.numel())


def make_case(q_lens, kv_lens, h, seed, kind="random", scale=SCALE_DSV3, extra_q=0):
    """q_lens[b] queries over kv_lens[b] keys for request b (kv_lens[b] - q_lens[b] is its prefix;
    negative: the first rows see no key)."""
    gen = torch.Generator().manual_seed(seed)
    tq, tkv = sum(q_lens), sum(kv_lens)
    rows = tkv + SLACK
    cu_q, cu_kv = _cu(q_lens), _cu(kv_lens)
    kv = torch.randn(rows, h, D_NOPE + DV, generator=gen, dtype=torch.float64)
    pe = torch.randn(rows, D_PE, generator=gen, dtype=torch.float64)
    q = torch.randn(tq, h, DQK, generator=gen, dtype=torch.float64)
    spread = 15.0  # std of s; the extremes of a row reach ~50
    if kind == "random":
        q *= spread / (math.sqrt(DQK) * scale)
    elif kind == "pe":
        q[..., :D_NOPE] = 0
        q *= spread / (math.sqrt(D_PE) * scale)
    else:
        freqs = torch.rand(D_NOPE // 2, generator=gen, dtype=torch.float64) * 0.8
        kv[:, :, :D_NOPE] = _codes(torch.arange(rows), freqs)[:, None, :]
        centers = torch.cat([int(cu_kv[b]) + kv_lens[b] - q_lens[b] + torch.arange(q_lens[b]) + 0.5
                             for b in range(len(q_lens))]) if tq else torch.zeros(0)
        q[..., :D_NOPE] = (EDGE_A / (D_NOPE // 2) / scale) * _codes(centers, freqs)[:, None, :]
        q[..., D_NOPE:] *= 1.0 / (math.sqrt(D_PE) * scale)
        for b in range(1, len(kv_lens)):
            if kv_lens[b] > 0:
                kv[int(cu_kv[b]), :, D_NOPE:] = POISON_V
    kv[tkv:] = math.nan
    pe[tkv:] = math.nan
    latent = torch.full((rows, 576), math.nan, dtype=torch.bfloat16)
    latent[:, 512:] = pe.to(torch.bfloat16)
    kv = kv.to(torch.bfloat16)
    return dict(q=q.to(torch.bfloat16), kv=kv, latent=latent, k_nope=kv[..., :D_NOPE],
                v=kv[..., D_NOPE:], k_pe=latent[:, 512:], cu_seqlens_q=cu_q, cu_seqlens_kv=cu_kv,
                max_q=max(q_lens) + extra_q, scale=scale, kind=kind, h=h, q_lens=list(q_lens),
                kv_lens=list(kv_lens))


def applicable(d, mutation):
    """Whether case `d` can show `mutation` at all."""
    pairs = [(nq, nk) for nq, nk in zip(d["q_lens"], d["kv_lens"]) if nq > 0]
    if mutation == "top_left":
        return any(nk > nq for nq, nk in pairs)
    if mutation in ("pe_per_head", "head_swap"):
        return d["h"] > 1
    if mutation == "kv_offset_from_q":
        return d["cu_seqlens_q"].tolist() != d["cu_seqlens_kv"].tolist()
    if mutation == "next_request_visible":
        return any(nk % 128 for _, nk in pairs)
    return True
