"""ORACLE — test infrastructure only (see oracle/__init__.py).

Absorbed MLA decode (csrc/decode_attn_mla.cu): an exact (fp64) reference with a per-element bound,
the lossy oracle of the two-part check, and restatements of kernel bugs (MUTATIONS).

Request b has n = kv_lens_total[b] cached tokens (the new ones included) and sq = mtp + 1 query
tokens; query row (sq_i, h) sees keys j <= n - sq + sq_i. With kv row k_j (576 wide),
s_j = (q . k_j) * softmax_scale and y = sum_j p_j k_j[:512] / L, p_j = exp(s_j - m), L = sum p_j.

The bound restates oracle/prefill_bf16.py's terms 1-7 (see its docstring) for this kernel:
  1. P rounding: bf16 of p against the running maximum, 2^-8 relative, ex2.approx flushes below
     2^-126; the row sum adds the unrounded values.
  2. Scores: one bf16 wgmma chain of 576 terms. The accumulation model (F16_ACC_EPS per 128 terms
     of the sum of magnitudes, oracle/moe_exact.py) scaled by the chain length: QK_EPS =
     F16_ACC_EPS * 576 / 128. Plus 2^-22 (|s| + |m|) for the fp32 scale constant and FMA, EXP_REL
     and one rescale (2^-21) per visited 64-key page.
  3. PV: O is one fp32 wgmma chain over the visited pages, 64 keys each:
     F16_ACC_EPS * n_pages * (1 + 2^-8) sum p|v| / L (an upper bound: a page is half a 128-term
     chain).
  4. fp32 bookkeeping: per page 16 additions per thread, the FMA into the running sum, the O
     rescale, a two-step quad sum, the IEEE 1 / L and O / L: (2 n_pages + 36) 2^-24 of sum p|v| / L.
  5. Output rounding to bf16: 2^-8 (|y| + B_rest).
  6. Split chunks store O_c = acc / L_c and lse_c = m_c + lg2.approx(L_c) (log2 units).
  7. Combine (mla_combine_kernel): M = max_c lse_c, w_c = ex2.approx(lse_c - M), one pass of
     fp32 FMAs, y = bf16(acc * (1 / l)). Per chunk weight: EXP_REL, the rounding of its argument
     (ln2 2^-23 Lam), lg2 (ln2 (2^-22 + 2^-24 Lam)); fp32: 2 roundings per chunk of acc and l and
     4 more: term_C = [2 e / (1 - e) + (2 C + 6) 2^-24] sum p|v| / L for pairs of C >= 2 chunks.

grade() / assert_exact() are oracle.attention_exact's two-part check.
"""
import math

import torch

from oracle.attention_exact import AGG_C, AGG_FLOOR, assert_exact, grade  # noqa: F401
from oracle.moe_exact import F16_ACC_EPS
from oracle.prefill_bf16 import EXP_REL, LG2_ABS, LN2

DQK = 576
DV = 512
PAGE = 64
ROWS = 64
QK_EPS = F16_ACC_EPS * DQK / 128
LOG2E = 1.0 / LN2

MUTATIONS = ("qk_512", "v_offset_64", "causal_off_by_one", "swap_pages", "tail_visible",
             "tile_row_shift", "mtp_rows_swapped", "scale_576", "chunk_dropped", "chunk_twice",
             "lse_natural_log", "o_half_repeated")


def num_tiles(h, sq):
    return (h * sq + ROWS - 1) // ROWS


def _combine_coef(s, vis, n_chunks):
    c = torch.as_tensor(n_chunks, dtype=torch.float64).reshape(-1, 1)
    smax = torch.where(vis, s.abs(), torch.zeros_like(s)).amax(1, keepdim=True)
    lam = smax * LOG2E + torch.log2(vis.sum(1, keepdim=True).clamp_min(1).double())
    e = torch.expm1(EXP_REL + LN2 * 2.0 ** -23 * lam + LN2 * (LG2_ABS + 2.0 ** -24 * lam))
    coef = 2 * e / (1 - e) + (2 * c + 6) * 2.0 ** -24
    return torch.where(c > 1, coef, torch.zeros_like(coef))


def _exact_rows(qr, kr, vr, vis, n_pages, scale, n_chunks):
    s = (qr @ kr.T) * scale
    s = torch.where(vis, s, torch.full_like(s, -math.inf))
    m = s.max(dim=1, keepdim=True).values
    p = torch.exp(s - m)
    L = p.sum(1, keepdim=True)
    y = (p @ vr) / L
    va, ya = vr.abs(), y.abs()
    nt = n_pages[:, None]
    delta = (QK_EPS * (qr.abs() @ kr.abs().T) * abs(scale) + 2.0 ** -22 * (s.abs() + m.abs())
             + EXP_REL + nt * 2.0 ** -21)
    delta = torch.where(vis, delta, torch.zeros_like(delta))
    r = torch.expm1(delta)
    lmin = L * torch.exp(-delta.max(dim=1, keepdim=True).values)
    pr = p * r
    phi_v = (p + pr) @ va
    term_s = (pr @ va + ya * pr.sum(1, keepdim=True)) / lmin
    term_p = (2.0 ** -8 * phi_v + 2.0 ** -126 * (vis.double() @ va)) / lmin
    term_pv = F16_ACC_EPS * nt * (1 + 2.0 ** -8) * phi_v / lmin
    term_f = (2 * nt + 36) * 2.0 ** -24 * phi_v / lmin
    term_c = _combine_coef(s, vis, n_chunks) * phi_v / lmin
    rest = term_s + term_p + term_pv + term_f + term_c
    return y, rest + 2.0 ** -8 * (ya + rest)


def _lossy_rows(qr, kr, vr, vis, scale, chunk_masks, mutation):
    """What the kernel computes with bf16 P, chunk by chunk (chunk_masks [C, N] bool), combined
    in log2 units; `mutation` restates one bug of the chunking or the combine."""
    s = (qr @ kr.T) * scale
    parts = []
    for cm in chunk_masks:
        v = vis & cm[None, :]
        sc = torch.where(v, s, torch.full_like(s, -math.inf))
        m = sc.max(dim=1, keepdim=True).values
        m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
        p = torch.exp(sc - m)
        L = p.sum(1, keepdim=True)
        o = (p.to(torch.bfloat16).double() @ vr) / L.clamp_min(1e-300)
        lse = torch.where(L > 0, m * LOG2E + torch.log2(L), torch.full_like(L, -math.inf))
        parts.append((o, lse))
    if mutation == "chunk_dropped" and len(parts) > 1:
        parts = parts[:-1]
    if mutation == "chunk_twice" and len(parts) > 1:
        parts = parts + parts[:1]
    if len(parts) == 1:
        return parts[0][0]
    lse = torch.cat([l for _, l in parts], 1)
    M = lse.max(1, keepdim=True).values
    w = torch.exp(lse - M) if mutation == "lse_natural_log" else torch.exp2(lse - M)
    acc = sum(w[:, i:i + 1] * parts[i][0] for i in range(len(parts)))
    return acc / w.sum(1, keepdim=True)


def _gather(kv, ids, n, pages_swapped=False):
    ids = ids.long().clone()
    if pages_swapped and ids.numel() >= 2:
        ids[[0, 1]] = ids[[1, 0]]
    return kv[ids].reshape(-1, kv.shape[2])[:n]


def mla_exact(q, kv, block_ids, kv_lens_total, num_seq_q, scale, chunks, lossy=False,
              mutation=None):
    """q [B*sq, H, 576], kv [blocks, 64, 576] (CPU, any float dtype), lengths include the new
    tokens; chunks = oracle.taskmap.pair_chunks(..., num_head_kv=T). Returns (y, B) float64
    [B*sq, H, 512]; lossy=True: (lossy oracle or mutant output, None)."""
    nb, h = kv_lens_total.numel(), q.shape[1]
    sq = num_seq_q
    T = num_tiles(h, sq)
    y = torch.full((nb * sq, h, DV), math.nan, dtype=torch.float64)
    bnd = torch.full_like(y, math.nan)
    for b in range(nb):
        n = int(kv_lens_total[b])
        npg = (n + PAGE - 1) // PAGE
        ids = block_ids[b, :npg]
        full = _gather(kv, ids, npg * PAGE, mutation == "swap_pages").double()
        k = full[:n]
        if mutation == "tail_visible":
            k = full
        kr = k.clone()
        if mutation == "qk_512":
            kr[:, DV:] = 0
        vr = k[:, :DV]
        if mutation == "v_offset_64":
            vr = k[:, 64:]
        N = k.shape[0]
        qb = q[b * sq:(b + 1) * sq].double().reshape(sq * h, DQK)  # row ri = sq_i * H + head
        ri = torch.arange(sq * h)
        if mutation == "tile_row_shift" and T > 1:
            qb = qb[(ri + ROWS) % (sq * h)]
        sqi = ri // h
        if mutation == "mtp_rows_swapped" and sq > 1:
            sqi = torch.where(sqi == 0, torch.ones_like(sqi), torch.where(sqi == 1, 0 * sqi, sqi))
        lim = n - sq + sqi + (1 if mutation == "causal_off_by_one" else 0)
        j = torch.arange(N)
        vis = (j[None, :] <= lim[:, None])
        if mutation != "tail_visible":
            vis &= j[None, :] < n
        sc = 1.0 / math.sqrt(DQK) if mutation == "scale_576" else scale
        tile_of = ri // ROWS
        nch = torch.tensor([len(chunks[(b, int(t))]) for t in tile_of], dtype=torch.float64)
        if lossy:
            out = torch.empty(sq * h, DV, dtype=torch.float64)
            for t in range(T):
                rows = tile_of == t
                cms = []
                for st, ln in chunks[(b, t)]:
                    cm = torch.zeros(N, dtype=torch.bool)
                    cm[st:st + ln] = True
                    if mutation == "tail_visible" and st + ln >= n:
                        cm[st:] = True
                    cms.append(cm)
                out[rows] = _lossy_rows(qb[rows], kr, vr, vis[rows], sc, cms, mutation)
            if mutation == "o_half_repeated":
                out[:, 256:] = out[:, :256]
            y[b * sq:(b + 1) * sq] = out.to(torch.bfloat16).double().reshape(sq, h, DV)
            continue
        npages = torch.full((sq * h,), float(npg), dtype=torch.float64)
        yy, bb = _exact_rows(qb, kr, vr, vis, npages, sc, nch)
        y[b * sq:(b + 1) * sq] = yy.reshape(sq, h, DV)
        bnd[b * sq:(b + 1) * sq] = bb.reshape(sq, h, DV)
    return (y, None) if lossy else (y, bnd)


def check(out, d, tag=""):
    """Two-part check of a kernel (or mutant) output against synth.attention_mla case `d`."""
    args = (d["q"], d["kv"], d["block_ids"], d["lens_total"], d["num_seq_q"], d["scale"],
            d["chunks"])
    exact, bound = mla_exact(*args)
    lossy, _ = mla_exact(*args, lossy=True)
    return grade(out, exact, bound, lossy)


def mutant(d, mutation):
    return mla_exact(d["q"], d["kv"], d["block_ids"], d["lens_total"], d["num_seq_q"], d["scale"],
                     d["chunks"], lossy=True, mutation=mutation)[0]
