"""Seeded inputs for the fused speculative sampler, and the same sampling as a torch chain.

`make_case` builds logits rows (synth/sampler.py families), a per-request temperature with greedy
and sampling requests mixed, drafts and uniforms planted so that each request accepts a chosen
number of drafts (all, none, all but the last, or any), and Gumbel noise. Every acceptance
decision clears a relative margin of MARGIN between fl(u q(d)) and p(d), and every emitting row's
winner beats its runner-up by MARGIN (fp64 keys, the residual made robust to a relative error
MARGIN in p): u or the row's noise is redrawn, and a request that 50 draws cannot clear makes the
builder raise. Planted cases: out-of-range drafts, p == q rows, q = 2 p rows (empty residual),
greedy argmax ties at the draft.

`torch_chain` is a vLLM-style rejection sampler written as torch ops; the benchmark times it and
the CPU tests compare it with the oracle.
"""
import zlib

import numpy as np
import torch

from oracle import sampler as osm, spec_sampler as osp
from synth import sampler as ss

MARGIN = 1e-4
FAMILIES = ("normal", "peaked", "ties")
OUT_OF_RANGE = (-1, -7)  # with V and V + 100


def _softmax64(xt_row):
    return osp._softmax64(xt_row[None].astype(np.float32))[0]


def _pick_accept(rng, p, q):
    """A draft token with p(d) / q(d) comfortably above 0 and its uniform: u q(d) < p(d)."""
    w = p * (q > 0) if q is not None else p
    d = int(rng.choice(p.size, p=w / w.sum())) if rng.uniform() < 0.7 else int(np.argmax(w))
    ratio = 1.0 if q is None else min(1.0, p[d] / q[d])
    if q is None:
        ratio = p[d]
    return d, np.float32(ratio * rng.uniform(0.02, 0.98))


def _pick_reject(rng, p, q, V):
    """A draft token that can be rejected (ratio p(d) / q(d) < 0.98) and its uniform."""
    if rng.uniform() < 0.25:
        d = int(rng.choice(OUT_OF_RANGE + (V, V + 100)))
        return d, np.float32(rng.uniform(0.05, 0.95))
    ratio = p if q is None else np.where(q > 0, p / np.maximum(q, 1e-38), np.inf)
    cand = np.nonzero(ratio < 0.98)[0]
    top = int(np.argmax(p))
    # the most likely token, when it can be rejected, is also the likely winner of the recovered
    # draw unless it is excluded
    d = top if ratio[top] < 0.98 and rng.uniform() < 0.4 else int(rng.choice(cand))
    r = float(ratio[d])
    return d, np.float32(r + (1 - r) * rng.uniform(0.05, 0.95))


def make_case(seed, B, K, V, dtype=torch.bfloat16, *, probs=False, forms="tensor", pad=0,
              draft_dtype=np.int64, families=FAMILIES):
    """One call: numpy inputs (`np`: store, V, drafts, draft_probs, temperature, uniform, noise),
    the logits storage [B (K + 1), V + pad] as a CPU tensor of `dtype` (`store_t`) and each
    request's planted number of accepted drafts (`plan`)."""
    rng = np.random.default_rng(seed)
    N = B * (K + 1)
    store, store_t, _ = ss.make_logits(rng, N, V, dtype, pad, 32, families)
    if forms == "tensor":
        temp = rng.choice(np.array([0.0, -1.0, np.nan, 0.7, 1.0, 1.5], np.float32), B)
    else:
        temp = np.float32(0.8)
    tt = np.broadcast_to(np.asarray(temp, np.float32), (B,))
    drafts = np.zeros((B, K), np.int64)
    uniform = rng.uniform(0.05, 0.95, (B, K)).astype(np.float32)
    qs = np.zeros((B, K, V), np.float32) if probs else None
    plan = np.zeros(B, np.int64)
    for b in range(B):
        n = [K, 0, K - 1, int(rng.integers(0, K + 1))][b % 4]
        plan[b] = n
        rows = slice(b * (K + 1), (b + 1) * (K + 1))
        x = store[rows, :V]
        if not tt[b] > 0:
            for i in range(K):
                a = osp.argmax_id(x[i])
                if b % 3 == 0 and i <= n and i < K:  # exact tie at the max: the smaller id wins
                    other = int(rng.integers(0, V))
                    if other != a:
                        store[b * (K + 1) + i, other] = store[b * (K + 1) + i, a]
                        x = store[rows, :V]
                        lo, hi = min(a, other), max(a, other)
                        drafts[b, i] = lo if i < n else hi
                        continue
                if i < n:
                    drafts[b, i] = a
                else:
                    drafts[b, i] = (a + 1 + int(rng.integers(0, V - 1))) % V if i == n else int(rng.integers(-2, V + 2))
            continue
        xt = (x / np.float32(tt[b])).astype(np.float32)
        for i in range(K):
            p = _softmax64(xt[i])
            q = None
            if probs:
                kind = rng.choice(["random", "random", "equal", "double"])
                if kind == "equal" and i == n:
                    kind = "random"  # p == q cannot reject
                if kind == "random":
                    qv = np.exp(rng.standard_normal(V) * 2.0)
                    qs[b, i] = (qv / qv.sum()).astype(np.float32)
                elif kind == "equal":
                    qs[b, i] = p.astype(np.float32)
                else:
                    qs[b, i] = (2 * p).astype(np.float32)  # q >= p everywhere: empty residual
                q = qs[b, i].astype(np.float64)
            if i < n:
                drafts[b, i], uniform[b, i] = _pick_accept(rng, p, q)
            elif i == n:
                drafts[b, i], uniform[b, i] = _pick_reject(rng, p, q, V)
            else:
                drafts[b, i] = int(rng.integers(-2, V + 2))
    # the row stores may have changed (planted ties): refresh the tensor
    store_t = torch.from_numpy(store).to(dtype)
    store = store_t.float().numpy()
    noise = ss.gumbel(rng, (N, V))
    kw = dict(draft_probs=qs, temperature=temp, uniform=uniform)
    for b in range(B):
        _clear_margins(rng, store, V, drafts, kw, noise, b)
    return dict(np=dict(store=store, V=V, draft_token_ids=drafts.astype(draft_dtype), noise=noise, **kw),
                store_t=store_t, plan=plan)


def request_detail(store, V, drafts, kw, noise, b):
    K = drafts.shape[1]
    rows = slice(b * (K + 1), (b + 1) * (K + 1))
    sub = dict(kw)
    sub["uniform"] = kw["uniform"][b:b + 1]
    if kw["draft_probs"] is not None:
        sub["draft_probs"] = kw["draft_probs"][b:b + 1]
    if isinstance(kw["temperature"], np.ndarray):
        sub["temperature"] = kw["temperature"][b:b + 1]
    # the request's rows keep their global row numbers for the noise
    n_all = np.zeros((K + 1, V), np.float32)
    n_all[:] = noise[rows]
    out, nacc, det = osp.spec_sample(store[rows], V, drafts[b:b + 1], noise=n_all, detail=True, **sub)
    return out[0], int(nacc[0]), det[0]


def request_ok(store, V, drafts, kw, noise, b):
    _, _, d = request_detail(store, V, drafts, kw, noise, b)
    return d["acc_margin"] >= MARGIN and d["gap"] >= MARGIN


def _clear_margins(rng, store, V, drafts, kw, noise, b, tries=50):
    K = drafts.shape[1]
    for _ in range(tries):
        _, _, d = request_detail(store, V, drafts, kw, noise, b)
        if d["acc_margin"] < MARGIN:  # move the uniforms away from the decision, keep the plan
            u = kw["uniform"][b]
            kw["uniform"][b] = np.clip(u * np.float32(rng.uniform(0.9, 1.1)), 2.0 ** -24, 1 - 2.0 ** -24)
            continue
        if d["gap"] < MARGIN:
            r = b * (K + 1) + d["n"]
            noise[r] = ss.gumbel(rng, V)
            continue
        return
    raise ValueError(f"synth.spec_sampler: request {b} stays within {MARGIN} of a rounding decision "
                     f"after {tries} draws")


def torch_chain(logits, draft_token_ids, draft_probs, temperature, uniform, noise):
    """vLLM-style rejection sampling as torch ops (fp32): softmax of x / t, acceptance u q(d) < p(d),
    the recovered token by Gumbel-max over max(0, p - q) (or, for one-hot drafts, over p without
    the draft), the bonus token by Gumbel-max over p; greedy requests compare drafts with the
    argmax. `temperature` is a [B] tensor. Returns (output_token_ids [B, K + 1], num_accepted [B])."""
    B, K = draft_token_ids.shape
    V = logits.shape[1]
    x = logits.float().view(B, K + 1, V)
    greedy = ~(temperature > 0)
    t = torch.where(greedy, torch.ones_like(temperature), temperature)
    xt = x / t[:, None, None]
    p = xt.softmax(-1)
    d = draft_token_ids.long()
    in_range = (d >= 0) & (d < V)
    dc = d.clamp(0, V - 1)
    g = noise.view(B, K + 1, V)
    if draft_probs is None:
        q = torch.zeros(B, K, V, device=logits.device).scatter_(-1, dc[..., None], 1.0)
    else:
        q = draft_probs
    pd = p[:, :K].gather(-1, dc[..., None])[..., 0]
    qd = q.gather(-1, dc[..., None])[..., 0]
    amax = x.argmax(-1)
    accept = torch.where(greedy[:, None], d == amax[:, :K], in_range & (uniform * qd < pd))
    n = accept.int().cumprod(-1).sum(-1)
    key = xt + g
    if draft_probs is None:
        rec = key[:, :K].scatter(-1, dc[..., None], float("-inf"))
        rec = torch.where(in_range[..., None], rec, key[:, :K])
    else:
        res = (p[:, :K] - q).clamp_min(0)
        rec = torch.where(res.sum(-1, keepdim=True) > 0, res.log() + g[:, :K], key[:, :K])
    cand = torch.cat([rec.argmax(-1), key[:, K:].argmax(-1)], -1)  # [B, K + 1]
    tok = torch.where(greedy, amax.gather(-1, n[:, None])[:, 0], cand.gather(-1, n[:, None])[:, 0])
    pos = torch.arange(K + 1, device=logits.device)[None]
    dd = torch.cat([d, torch.zeros_like(d[:, :1])], -1)
    out = torch.where(pos < n[:, None], dd, torch.where(pos == n[:, None], tok[:, None], -1))
    return out.int(), n.int()


# The GPU test's grid: (dtype, B, K, V, probs, forms)
BIG_V = (120832, 151936)
GRID = (
    [(dt, 4, K, 4096, pr, "tensor") for dt in ("fp32", "bf16") for K in (1, 2, 3, 4, 8) for pr in (False, True)]
    + [(dt, B, 2, V, pr, "tensor") for dt in ("fp32", "bf16") for B in (1, 64) for V in BIG_V
       for pr in (False, True)]
    + [(dt, 64, 3, 151936, pr, "scalar") for dt in ("fp32", "bf16") for pr in (False, True)]
    + [("bf16", 16, 8, 151936, True, "tensor"), ("bf16", 512, 1, 120832, False, "tensor"),
       ("bf16", 512, 1, 4096, True, "tensor"), ("fp32", 512, 3, 4096, False, "tensor")]
)


def _seed(*key):
    return zlib.crc32(repr(key).encode()) % 100003


def case(dt, B, K, V, probs, forms):
    """The GRID case: +inf row padding of 4 or 256 (fp32, odd / even B) or 128 (bf16); int32 drafts
    for odd B, int64 for even B."""
    pad = (4 if B % 2 else 256) if dt == "fp32" else 128
    return make_case(_seed(dt, B, K, V, probs, forms), B, K, V,
                     dtype=torch.float32 if dt == "fp32" else torch.bfloat16, probs=probs, forms=forms,
                     pad=pad, draft_dtype=np.int32 if B % 2 else np.int64)
