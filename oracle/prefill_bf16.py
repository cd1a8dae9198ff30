"""ORACLE — test infrastructure only (see oracle/__init__.py).

BF16 causal prefill: torch restatements of the reference's ground truth, and an exact (fp64)
reference with a per-element error bound for the kernel (csrc/prefill_bf16.cu).

Restatements (pinned by tests/golden/prefill_bf16_*.npz, which
tests/golden/make_golden_prefill_bf16.py makes by running the reference's own functions on CPU):
  varlen_prefill   reference tests/test_attention_prefill_bf16.py `naive_attn_varlen_func`
                   (causal, cu_seqlens_k = cu_seqlens_q, GQA by repeating kv heads)
  kvcache_prefill  reference tests/test_attention_with_kvcache_prefill_bf16.py
                   `naive_attn_with_kvcache_func`, generalised to ragged and chunked requests
                   (request b: sq = cu_seqlens_q[b+1] - cu_seqlens_q[b] new tokens, the last of its
                   skv = seqlens_kv[b] cached ones; sq = 0 writes nothing).

Exact check (notation of oracle/attention_exact.py, one query row, natural-log units): over the
visible keys j, s_j = q.k_j / sqrt(128), m = max s_j, p_j = exp(s_j - m), L = sum p_j,
y = sum p_j v_j / L. What the kernel computes differently:

1. P rounding. P goes to the PV wgmma as bf16 of p~ = 2^(s log2e - r), r the running maximum
   (<= m): round-to-nearest-even with 8 significant bits is within 2^-8 of p~ relative, which
   stays 2^-8 of p in units of the true maximum. ex2.approx.ftz flushes results below 2^-126 to 0.
       term_P = (2^-8 sum p_j |v_j| + 2^-126 sum_vis |v_j|) / L
   The row sum adds the unrounded values, so P rounding enters the numerator only.
2. Score and exponential error, entering numerator and row sum alike (bounded as in
   attention_exact: r_j <= expm1(delta_j), denominator >= L exp(-max delta)):
       delta_j = F16_ACC_EPS * sum_i |q_i k_ji| / sqrt(128)   (bf16 wgmma, one 128-term chain)
               + 2^-22 (|s_j| + |m|)                          (fp32 scale constant and FMA)
               + EXP_REL + n_tiles 2^-21                      (ex2.approx; one rescale per tile)
   F16_ACC_EPS is the accumulation model of oracle/moe_exact.py (a model, not a derivation:
   an fp32 adder that truncates, at most 2^-16 of the sum of magnitudes per 128 terms).
3. PV accumulation: O is one fp32 wgmma chain over all n_tiles visited 128-key tiles:
       term_PV = F16_ACC_EPS * n_tiles * (1 + 2^-8) sum p_j |v_j| / L
4. fp32 bookkeeping: the per-tile O rescale (n_tiles products), the row sum ((34 + n_tiles)
   additions of positive terms), 1 / L and O / L: (n_tiles + 34 + n_tiles + 2) 2^-24 of
   sum p_j |v_j| / L.
5. Output rounding to bf16: 2^-8 (|y| + B_rest).

grade() / assert_exact() are oracle.attention_exact's two-part check: (a) |kernel - exact| <= B
element-wise, (b) rel L2 of the kernel within AGG_C times that of the lossy oracle (P rounded to
bf16 as the kernel rounds it, against the row maximum) plus AGG_FLOOR.

MUTATIONS are the kernel bugs the tests show the check detects; each restates the oracle with
one mistake (see _request).
"""
import math

import torch

from oracle.attention_exact import AGG_C, AGG_FLOOR, assert_exact, grade  # noqa: F401
from oracle.moe_exact import F16_ACC_EPS

D = 128
TILE = 128
EXP_REL = 2.0 ** -22 + 2.0 ** -21  # ex2.approx.ftz.f32 (PTX ISA: 2^-22 relative), plus headroom
MUTATIONS = ("top_left", "causal_off_by_one", "kv_head_mod", "swap_pages", "tail_visible",
             "v_shift", "dense_prev_offset", "no_scale")


# ------------------------------------------------------------------------------------------------
# restatements of the reference's ground truth (fp32 math)
# ------------------------------------------------------------------------------------------------
def varlen_prefill(q, k, v, cu_seqlens_q):
    """q [total, Hq, D], k/v [total, Hkv, D] (on any device); causal per request. Returns float32
    [total, Hq, D] (rows of no request stay 0)."""
    g = q.shape[1] // k.shape[1]
    out = torch.zeros(q.shape, dtype=torch.float32, device=q.device)
    for b in range(cu_seqlens_q.numel() - 1):
        s0, s1 = int(cu_seqlens_q[b]), int(cu_seqlens_q[b + 1])
        if s1 == s0:
            continue
        qi = q[s0:s1].float()
        ki = k[s0:s1].float().repeat_interleave(g, 1)
        vi = v[s0:s1].float().repeat_interleave(g, 1)
        scores = torch.einsum("qhd,khd->hqk", qi, ki) / math.sqrt(q.shape[2])
        mask = torch.triu(torch.ones(s1 - s0, s1 - s0, device=q.device), diagonal=1).bool()
        scores.masked_fill_(mask, float("-inf"))
        out[s0:s1] = torch.einsum("hqk,khd->qhd", torch.softmax(scores, -1), vi)
    return out


def gather_pages(cache, ids, n):
    """Tokens 0..n-1 of a request from its pages: [n, Hkv, D]."""
    return cache[ids.long()].reshape(-1, cache.shape[2], cache.shape[3])[:n]


def kvcache_prefill(q, kcache, vcache, cu_seqlens_q, block_ids, seqlens_kv):
    """q [total, Hq, D]; caches [blocks, bs, Hkv, D]. Returns float32 [total, Hq, D]."""
    bs, hkv = kcache.shape[1], kcache.shape[2]
    g = q.shape[1] // hkv
    out = torch.zeros(q.shape, dtype=torch.float32, device=q.device)
    for b in range(seqlens_kv.numel()):
        s0, s1 = int(cu_seqlens_q[b]), int(cu_seqlens_q[b + 1])
        nq, nkv = s1 - s0, int(seqlens_kv[b])
        if nq == 0:
            continue
        ids = block_ids[b, :(nkv + bs - 1) // bs]
        bq = q[s0:s1].transpose(0, 1).float()
        bk = gather_pages(kcache, ids, nkv).transpose(0, 1).repeat_interleave(g, 0).float()
        bv = gather_pages(vcache, ids, nkv).transpose(0, 1).repeat_interleave(g, 0).float()
        scores = bq @ bk.transpose(-2, -1) / math.sqrt(q.shape[2])
        cm = torch.tril(torch.ones(nkv, nkv, dtype=torch.bool, device=q.device))[nkv - nq:, :]
        scores = scores.masked_fill(~cm, float("-inf"))
        out[s0:s1] = (torch.softmax(scores, -1) @ bv).transpose(0, 1)
    return out


# ------------------------------------------------------------------------------------------------
# exact reference, bound, lossy oracle
# ------------------------------------------------------------------------------------------------
def _rows(qr, kr, vr, vis, n_tiles, scale, lossy):
    """One (request, q head) in fp64: qr [R, D], kr / vr [N, D], vis [R, N] bool, n_tiles [R].
    Returns (y, B), or the lossy oracle's y (bf16-rounded P), [R, D]; NaN rows see no key."""
    s = (qr @ kr.T) * scale
    s = torch.where(vis, s, torch.full_like(s, -math.inf))
    m = s.max(dim=1, keepdim=True).values
    dead = ~torch.isfinite(m)
    m = torch.where(dead, torch.zeros_like(m), m)
    p = torch.exp(s - m)
    L = p.sum(1, keepdim=True)
    nan = torch.full((qr.shape[0], vr.shape[1]), math.nan, dtype=torch.float64)
    if lossy:
        y = (p.to(torch.bfloat16).double() @ vr) / L
        return torch.where(dead, nan, y.to(torch.bfloat16).double()), None
    y = (p @ vr) / L
    va, ya = vr.abs(), y.abs()
    visf = vis.double()
    nt = n_tiles[:, None]
    delta = (F16_ACC_EPS * (qr.abs() @ kr.abs().T) * abs(scale) + 2.0 ** -22 * (s.abs() + m.abs())
             + EXP_REL + nt * 2.0 ** -21)
    delta = torch.where(vis, delta, torch.zeros_like(delta))
    r = torch.expm1(delta)
    lmin = L * torch.exp(-delta.max(dim=1, keepdim=True).values)
    pr = p * r
    phi_v = (p + pr) @ va
    term_s = (pr @ va + ya * pr.sum(1, keepdim=True)) / lmin
    term_p = (2.0 ** -8 * phi_v + 2.0 ** -126 * (visf @ va)) / lmin
    term_pv = F16_ACC_EPS * nt * (1 + 2.0 ** -8) * phi_v / lmin
    term_f = (2 * nt + 36) * 2.0 ** -24 * phi_v / lmin
    rest = term_s + term_p + term_pv + term_f
    bound = rest + 2.0 ** -8 * (ya + rest)
    return torch.where(dead, nan, y), torch.where(dead, nan, bound)


def _request(qb, kb, vb, nq, nkv, hq_count, lossy, mutation, page):
    """All q heads of one request. qb [nq, Hq, D]; kb / vb [>= nkv, Hkv, D] (rows past nkv: the
    rest of the last page, read only by the tail_visible mutation). Returns (y, B) [nq, Hq, D]."""
    hkv = kb.shape[1]
    g = hq_count // hkv
    scale = 1.0 / math.sqrt(D)
    n_eff = nkv
    if mutation == "tail_visible":  # length rounded up to whole pages, causal limit included
        n_eff = (nkv + page - 1) // page * page
    if mutation == "swap_pages" and nkv > page:  # the request's last two pages exchanged
        last = (nkv - 1) // page
        idx = torch.arange(kb.shape[0])
        a, b = torch.arange((last - 1) * page, last * page), torch.arange(last * page, (last + 1) * page)
        b = b[b < kb.shape[0]]
        idx[a[:b.numel()]], idx[b] = b, a[:b.numel()]
        kb, vb = kb[idx], vb[idx]
    if mutation == "v_shift":  # V read one token late
        vb = torch.cat([vb[1:], vb[-1:]])
    if mutation == "no_scale":
        scale = 1.0
    pos = torch.arange(n_eff)
    row = torch.arange(nq)
    lim = n_eff - nq + row
    if mutation == "top_left":
        lim = row
    elif mutation == "causal_off_by_one":
        lim = lim + 1
    vis = (pos[None, :] <= lim[:, None]) & (pos[None, :] < n_eff)
    # tiles the kernel visits for each row's 128-row Q tile (prefill_common.cuh decode_work)
    tile_hi = torch.clamp(nkv - nq + (row // TILE + 1) * TILE, 0, nkv)
    n_tiles = ((tile_hi + TILE - 1) // TILE).double()
    y = torch.empty(nq, hq_count, D, dtype=torch.float64)
    bound = torch.empty_like(y)
    for h in range(hq_count):
        hk = h % hkv if mutation == "kv_head_mod" else h // g
        yr, br = _rows(qb[:, h].double(), kb[:n_eff, hk].double(), vb[:n_eff, hk].double(), vis,
                       n_tiles, scale, lossy)
        y[:, h] = yr
        if br is not None:
            bound[:, h] = br
    return y, bound


def _run(q, source, cu_seqlens_q, lossy, mutation, page):
    total, hq, _ = q.shape
    y = torch.full((total, hq, D), math.nan, dtype=torch.float64)
    bound = torch.full_like(y, math.nan)
    for b in range(cu_seqlens_q.numel() - 1):
        s0, s1 = int(cu_seqlens_q[b]), int(cu_seqlens_q[b + 1])
        if s1 == s0:
            continue
        kb, vb, nkv = source(b)
        yr, br = _request(q[s0:s1], kb, vb, s1 - s0, nkv, hq, lossy, mutation, page)
        y[s0:s1], bound[s0:s1] = yr, br
    return y, bound


def dense_exact(q, k, v, cu_seqlens_q, lossy=False, mutation=None):
    """attention_prefill_bf16 on CPU tensors. Returns (y, B) float64 [total, Hq, D]; with
    lossy=True the first is the lossy oracle's output. Rows of no request are NaN."""
    cu = cu_seqlens_q

    def source(b):
        s0, s1 = int(cu[b]), int(cu[b + 1])
        if mutation == "dense_prev_offset" and b > 0:
            s0, s1 = int(cu[b - 1]), int(cu[b - 1]) + (s1 - s0)
        return k[s0:s1], v[s0:s1], s1 - s0

    return _run(q, source, cu, lossy, mutation, TILE)


def paged_exact(q, kcache, vcache, cu_seqlens_q, block_ids, seqlens_kv, lossy=False,
                mutation=None):
    """attention_with_kvcache_prefill_bf16. Returns (y, B) float64 [total, Hq, D]."""
    bs = kcache.shape[1]

    def source(b):
        nkv = int(seqlens_kv[b])
        nblk = (nkv + bs - 1) // bs
        ids = block_ids[b, :nblk]
        return gather_pages(kcache, ids, nblk * bs), gather_pages(vcache, ids, nblk * bs), nkv

    return _run(q, source, cu_seqlens_q, lossy, mutation, bs)


def check(out, d, mutation=None, tag=""):
    """Grades a kernel output (or a mutant) against the exact reference of synth input `d`
    (synth.prefill_bf16.make_exact_case). Returns grade()'s dict."""
    if d["op"] == "dense":
        exact, bound = dense_exact(d["q"], d["k"], d["v"], d["cu_seqlens_q"])
        lossy, _ = dense_exact(d["q"], d["k"], d["v"], d["cu_seqlens_q"], lossy=True)
    else:
        args = (d["q"], d["kcache"], d["vcache"], d["cu_seqlens_q"], d["block_ids"], d["seqlens_kv"])
        exact, bound = paged_exact(*args)
        lossy, _ = paged_exact(*args, lossy=True)
    return grade(out, exact, bound, lossy)


def mutant(d, mutation):
    """What a kernel with `mutation` would compute on synth input `d` (bf16 P, bf16 output)."""
    if d["op"] == "dense":
        return dense_exact(d["q"], d["k"], d["v"], d["cu_seqlens_q"], lossy=True,
                           mutation=mutation)[0]
    return paged_exact(d["q"], d["kcache"], d["vcache"], d["cu_seqlens_q"], d["block_ids"],
                       d["seqlens_kv"], lossy=True, mutation=mutation)[0]
