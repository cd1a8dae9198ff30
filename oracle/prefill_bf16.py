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

BF16 paged decode (csrc/decode_attn_bf16.cu, decode_exact) is this computation with
cu_seqlens_q = sq * arange(B + 1): request b has sq = mtp + 1 query rows and row i sees keys
<= n_b - sq + i. Its QK chain, log2-domain online softmax with ex2.approx, bf16 P against a
running maximum <= the row maximum, bf16 PV wgmma and fp32 rescales are the prefill's, so terms
1-5 apply, with two differences:

6. Tiles and PV chains. Decode splits a (request, kv head) pair into split-k chunks of whole
   128-key tiles (oracle.taskmap), keeps the running maximum per chunk and starts a fresh PV
   wgmma chain per tile. A chunk's maximum is <= the row maximum, so terms 1-2 hold in units of
   the true maximum as they stand; a chunk visits at most n_tiles tiles of the request, so
   n_tiles 2^-21 (rescales) and n_tiles 2^-24 (O rescales) are upper bounds; and the PV error of
   per-tile chains is at most F16_ACC_EPS times the sum of the tiles' magnitudes, which
   F16_ACC_EPS n_tiles sum p|v| / L bounds. The per-chunk row sum takes one FMA per tile per
   lane, a 5-level warp sum and 3 additions across warps (n_tiles + 8 roundings), 26 fewer than
   term 4 allots; that covers the 1 ulp (2^-23) of rcp.approx in O * rcp.approx(L).
   A pair with one chunk writes bf16(O * rcp.approx(L)) from the attention kernel: terms 1-6.
7. Split-k combine (decode_combine_kernel, csrc/decode_attn_fp8.cu), pairs of C >= 2 chunks. Each
   chunk stores O_c = acc * rcp.approx(tot) (counted in 6) and lse_c = m_c + lg2.approx(tot) in
   log2 units. The combine runs C / 4 chunks per warp: w = ex2.approx(lse_c - m), the running
   rescale ex2.approx(m - m_new) of acc and l, then one ex2.approx(m_w - m_g) per warp when the
   four warps merge; y = bf16((sum w O_c) * (1 / sum w)), the division IEEE (no fast-math).
   With Lam = log2(e) max_vis |s_j| + log2(n_vis) >= |lse_c| (and >= |m_c log2 e|):
     - lg2.approx: absolute error <= 2^-22 (PTX ISA: 2^-22.6 on the mantissa); rounding of
       m_c + lg2: <= 2^-24 Lam. Weight error ln2 (2^-22 + 2^-24 Lam), relative.
     - every ex2.approx that scales chunk c's weight (at most ceil(C/4) + 1 of them): EXP_REL,
       plus the rounding of its argument, |x| <= 2 Lam: ln2 2^-23 Lam.
     - a relative weight error e moves y by |sum_c w_c e_c (O_c - y)| / sum_c w_c (1 + e_c)
       <= 2 e / (1 - e) sum p|v| / L (sum_c w_c |O_c| <= sum p|v|, |y| <= sum p|v| / L).
     - fp32 arithmetic: at most 3 roundings per chunk step of acc and of l, 4 more in the warp
       merge of each, then 1 / l and the product: (6 ceil(C/4) + 10) 2^-24 of sum p|v| / L.
   term_C = [2 e / (1 - e) + (6 ceil(C/4) + 10) 2^-24] sum p|v| / L, with
   e = expm1((ceil(C/4) + 1)(EXP_REL + ln2 2^-23 Lam) + ln2 (2^-22 + 2^-24 Lam)).
   The FP8 oracle's flat 2^-20 for this step (oracle/attention_exact.py term 4) does not hold in
   general: the fp32 operations alone reach 2^-20 at C = 2, and the weight errors grow with Lam
   and C. Here the term is evaluated per row from the pair's chunk count.

MUTATIONS are the prefill kernel bugs the tests show the check detects and DECODE_MUTATIONS the
decode ones; each restates the oracle with one mistake (see _request).
"""
import math

import torch

from oracle.attention_exact import AGG_C, AGG_FLOOR, assert_exact, grade  # noqa: F401
from oracle.moe_exact import F16_ACC_EPS

D = 128
TILE = 128
EXP_REL = 2.0 ** -22 + 2.0 ** -21  # ex2.approx.ftz.f32 (PTX ISA: 2^-22 relative), plus headroom
LG2_ABS = 2.0 ** -22               # lg2.approx.f32 (PTX ISA: 2^-22.6 absolute on the mantissa)
LN2 = math.log(2.0)
MUTATIONS = ("top_left", "causal_off_by_one", "kv_head_mod", "swap_pages", "tail_visible",
             "v_shift", "dense_prev_offset", "no_scale")
# decode: the shared ones, then bugs of the page walk, the MTP rows and the split-k combine
DECODE_MUTATIONS = ("causal_off_by_one", "top_left", "tail_visible", "swap_pages",
                    "swap_first_pages", "v_shift", "kv_head_mod", "q_heads_reversed",
                    "mtp_rows_swapped", "no_scale", "page_group_wrap", "chunk_dropped",
                    "chunk_twice", "lse_natural_log")


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
def _combine_coef(s, vis, n_chunks):
    """Term 7 per row, in units of sum p|v| / L: [R, 1], 0 where the pair has one chunk."""
    c = torch.as_tensor(n_chunks, dtype=torch.float64).reshape(-1, 1)
    per_warp = torch.ceil(c / 4)
    smax = torch.where(vis, s.abs(), torch.zeros_like(s)).amax(1, keepdim=True)
    lam = smax / LN2 + torch.log2(vis.sum(1, keepdim=True).clamp_min(1).double())
    e = torch.expm1((per_warp + 1) * (EXP_REL + LN2 * 2.0 ** -23 * lam)
                    + LN2 * (LG2_ABS + 2.0 ** -24 * lam))
    coef = 2 * e / (1 - e) + (6 * per_warp + 10) * 2.0 ** -24
    return torch.where(c > 1, coef, torch.zeros_like(coef))


def _rows(qr, kr, vr, vis, n_tiles, scale, lossy, n_chunks=1, bias=None):
    """One (request, q head) in fp64: qr [R, D], kr / vr [N, D], vis [R, N] bool, n_tiles [R],
    n_chunks: split-k chunks of the row's (request, kv head) pair (decode), bias [R, N]: added to
    the scores (mutants only). Returns (y, B), or the lossy oracle's y (bf16-rounded P), [R, D];
    NaN rows see no key."""
    s = (qr @ kr.T) * scale
    if bias is not None:
        s = s + bias
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
    term_c = _combine_coef(s, vis, n_chunks) * phi_v / lmin
    rest = term_s + term_p + term_pv + term_f + term_c
    bound = rest + 2.0 ** -8 * (ya + rest)
    return torch.where(dead, nan, y), torch.where(dead, nan, bound)


def _chunk_keys(chunk, n):
    st, ln = chunk
    return torch.arange(st, min(st + ln, n))


def _decode_head_mutation(mutation, chunks, qr, kr, vis, scale, page, n):
    """Key source index [n] and score bias [R, n] (or None) of a decode mutation for one q head
    whose kv head's pair is split into `chunks` [(start, length)] (oracle.taskmap.pair_chunks)."""
    src = torch.arange(n)
    bias = None
    if mutation == "page_group_wrap":  # page ids of a chunk fetched only for its first 32 pages
        for st, ln in chunks:
            j = _chunk_keys((st, ln), n)
            rel = j - st
            src[j] = st + (rel // page % 32) * page + rel % page
    elif mutation in ("chunk_dropped", "chunk_twice", "lse_natural_log") and len(chunks) > 1:
        bias = torch.zeros(qr.shape[0], n, dtype=torch.float64)
        if mutation == "chunk_dropped":  # the combine skips chunk 1
            bias[:, _chunk_keys(chunks[1], n)] = -math.inf
        elif mutation == "chunk_twice":  # chunk 0 added twice
            bias[:, _chunk_keys(chunks[0], n)] = LN2
        else:  # lse = m + ln(tot) read as log2: chunk weight tot^ln2 instead of tot
            s = torch.where(vis, (qr @ kr.T) * scale, torch.full_like(bias, -math.inf))
            for ch in chunks:
                j = _chunk_keys(ch, n)
                sc = s[:, j]
                mc = sc.max(1, keepdim=True).values
                live = torch.isfinite(mc)
                tot = torch.exp(sc - torch.where(live, mc, torch.zeros_like(mc))).sum(1, keepdim=True)
                bias[:, j] = torch.where(live, (LN2 - 1) * torch.log(tot.clamp_min(1e-300)),
                                         torch.zeros_like(tot))
    return src, bias


def _request(qb, kb, vb, nq, nkv, hq_count, lossy, mutation, page, chunks=None):
    """All q heads of one request. qb [nq, Hq, D]; kb / vb [>= nkv, Hkv, D] (rows past nkv: the
    rest of the last page, read only by the tail_visible mutation); chunks (decode): kv head ->
    its split-k chunks [(start, length)]. Returns (y, B) [nq, Hq, D]."""
    hkv = kb.shape[1]
    g = hq_count // hkv
    scale = 1.0 / math.sqrt(D)
    n_eff = nkv
    if mutation == "tail_visible":  # length rounded up to whole pages, causal limit included
        n_eff = (nkv + page - 1) // page * page
    if mutation == "causal_off_by_one" and chunks is not None and nkv % page:
        n_eff = nkv + 1  # decode: length + 1, every row sees one more key
    if mutation in ("swap_pages", "swap_first_pages") and nkv > page:
        # the request's last two pages exchanged, or its first two (one 128-key tile)
        last = (nkv - 1) // page if mutation == "swap_pages" else 1
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
    elif mutation == "mtp_rows_swapped":  # row i masked as row nq - 1 - i
        lim = n_eff - 1 - row
    vis = (pos[None, :] <= lim[:, None]) & (pos[None, :] < n_eff)
    # tiles the kernel visits for each row's 128-row Q tile (prefill_common.cuh decode_work)
    tile_hi = torch.clamp(nkv - nq + (row // TILE + 1) * TILE, 0, nkv)
    n_tiles = ((tile_hi + TILE - 1) // TILE).double()
    y = torch.empty(nq, hq_count, D, dtype=torch.float64)
    bound = torch.empty_like(y)
    for h in range(hq_count):
        hk = h % hkv if mutation == "kv_head_mod" else h // g
        hqs = hk * g + (g - 1 - h % g) if mutation == "q_heads_reversed" else h
        qr, kr, vr = qb[:, hqs].double(), kb[:n_eff, hk].double(), vb[:n_eff, hk].double()
        nch, bias = 1, None
        if chunks is not None:
            ch = chunks[h // g]
            nch = len(ch)
            src, bias = _decode_head_mutation(mutation, ch, qr, kr, vis, scale, page, n_eff)
            kr, vr = kr[src], vr[src]
        yr, br = _rows(qr, kr, vr, vis, n_tiles, scale, lossy, nch, bias)
        y[:, h] = yr
        if br is not None:
            bound[:, h] = br
    return y, bound


def _run(q, source, cu_seqlens_q, lossy, mutation, page, chunks=None):
    total, hq, _ = q.shape
    y = torch.full((total, hq, D), math.nan, dtype=torch.float64)
    bound = torch.full_like(y, math.nan)
    for b in range(cu_seqlens_q.numel() - 1):
        s0, s1 = int(cu_seqlens_q[b]), int(cu_seqlens_q[b + 1])
        if s1 == s0:
            continue
        kb, vb, nkv = source(b)
        ch = None if chunks is None else {h: chunks[(b, h)] for h in range(kb.shape[1])}
        yr, br = _request(q[s0:s1], kb, vb, s1 - s0, nkv, hq, lossy, mutation, page, ch)
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
                mutation=None, chunks=None):
    """attention_with_kvcache_prefill_bf16 (chunks None) or, with chunks = the split-k chunks of
    every (request, kv head) pair (oracle.taskmap.pair_chunks), bf16 paged decode. Returns (y, B)
    float64 [total, Hq, D]."""
    bs = kcache.shape[1]

    def source(b):
        nkv = int(seqlens_kv[b])
        nblk = (nkv + bs - 1) // bs
        ids = block_ids[b, :nblk]
        return gather_pages(kcache, ids, nblk * bs), gather_pages(vcache, ids, nblk * bs), nkv

    return _run(q, source, cu_seqlens_q, lossy, mutation, bs, chunks)


def decode_exact(q, kcache, vcache, block_ids, kv_lens_total, num_seq_q, chunks, lossy=False,
                 mutation=None):
    """attention_decode_bf16 (lengths include the num_seq_q new tokens) on CPU tensors, scheduled
    as `chunks` describes (oracle.taskmap.pair_chunks). Returns (y, B) float64 [B*sq, Hq, D]; with
    lossy=True the first is the lossy oracle's output (or a mutant's)."""
    cu = num_seq_q * torch.arange(kv_lens_total.numel() + 1)
    return paged_exact(q, kcache, vcache, cu, block_ids, kv_lens_total, lossy, mutation, chunks)


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
