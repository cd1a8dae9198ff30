"""ORACLE — test infrastructure only (see oracle/__init__.py).

MLA prefill (csrc/prefill_mla.cu): an exact (fp64) reference with a per-element bound, the lossy
oracle of the two-part check, and restatements of kernel bugs (MUTATIONS).

Request b has nq = cu_seqlens_q[b+1] - cu_seqlens_q[b] queries and nk = cu_seqlens_kv[b+1] -
cu_seqlens_kv[b] keys, at key rows kv0 = cu_seqlens_kv[b] ..; query i sees keys j <= nk - nq + i.
For head h, key j is [k_nope[kv0 + j, h] (128) | k_pe[kv0 + j] (64)], its value v[kv0 + j, h] (128),
and s_j = (q . k_j) * softmax_scale.

The bound restates oracle/prefill_bf16.py's terms 1-5 (see its docstring) for this kernel:
  1. P rounding: bf16 of p against the running maximum, 2^-8 relative; ex2.approx flushes below
     2^-126. The row sum adds the unrounded values.
  2. Scores: one bf16 wgmma chain of 192 terms, QK_EPS = F16_ACC_EPS * 192 / 128 of the sum of
     magnitudes (the accumulation model of oracle/moe_exact.py scaled by the chain length), plus
     2^-22 (|s| + |m|) for the fp32 scale constant (log2e * softmax_scale rounded once) and the
     FMA, EXP_REL, and one rescale (2^-21) per visited 128-key tile.
  3. PV: one fp32 wgmma chain over the visited tiles: F16_ACC_EPS n_tiles (1 + 2^-8) sum p|v| / L.
  4. fp32 bookkeeping: (2 n_tiles + 36) 2^-24 of sum p|v| / L.
  5. Output rounding to bf16: 2^-8 (|y| + B_rest).
n_tiles is the count of 128-key tiles the row's 128-row Q tile visits (prefill_common.cuh
decode_work). A row that sees no key (nk < nq) is written as exact zeros: y = 0, B = 0.

The reference is computed on whatever device its inputs are on (fp64 throughout), so a GPU test
can evaluate it for long requests; `rows` restricts it to a subset of query rows.

grade() / assert_exact() are oracle.attention_exact's two-part check.
"""
import math

import torch

from oracle.attention_exact import AGG_C, AGG_FLOOR, assert_exact, grade  # noqa: F401
from oracle.moe_exact import F16_ACC_EPS
from oracle.prefill_bf16 import EXP_REL

D_NOPE = 128
D_PE = 64
DQK = D_NOPE + D_PE
DV = 128
TILE = 128
QK_EPS = F16_ACC_EPS * DQK / 128
_BUDGET = 1 << 24  # fp64 elements of one [H, rows, keys] intermediate

MUTATIONS = ("top_left", "causal_off_by_one", "pe_dropped", "pe_per_head", "kv_offset_from_q",
             "next_request_visible", "v_from_k_nope", "head_swap", "scale_ignored")


def _rows(qr, kr, vr, vis, n_tiles, scale, lossy):
    """All heads of a block of query rows in fp64: qr [H, R, 192], kr [H, N, 192], vr [H, N, 128],
    vis [R, N] bool, n_tiles [R]. Returns (y, B) [H, R, 128]; lossy: (bf16-P oracle output, None).
    Rows that see no key are 0 with B = 0."""
    s = (qr @ kr.transpose(1, 2)) * scale
    s = torch.where(vis, s, torch.full_like(s, -math.inf))
    m = s.amax(2, keepdim=True)
    dead = ~torch.isfinite(m)
    m = torch.where(dead, torch.zeros_like(m), m)
    p = torch.exp(s - m)
    L = p.sum(2, keepdim=True)
    zero = torch.zeros((), dtype=torch.float64, device=qr.device)
    if lossy:
        y = (p.to(torch.bfloat16).double() @ vr) / L
        return torch.where(dead, zero, y.to(torch.bfloat16).double()), None
    y = (p @ vr) / L
    va, ya = vr.abs(), y.abs()
    nt = n_tiles[None, :, None]
    delta = (QK_EPS * (qr.abs() @ kr.abs().transpose(1, 2)) * abs(scale)
             + 2.0 ** -22 * (s.abs() + m.abs()) + EXP_REL + nt * 2.0 ** -21)
    delta = torch.where(vis, delta, torch.zeros_like(delta))
    r = torch.expm1(delta)
    lmin = L * torch.exp(-delta.amax(2, keepdim=True))
    pr = p * r
    phi_v = (p + pr) @ va
    term_s = (pr @ va + ya * pr.sum(2, keepdim=True)) / lmin
    term_p = (2.0 ** -8 * phi_v + 2.0 ** -126 * (vis.double() @ va)) / lmin
    term_pv = F16_ACC_EPS * nt * (1 + 2.0 ** -8) * phi_v / lmin
    term_f = (2 * nt + 36) * 2.0 ** -24 * phi_v / lmin
    rest = term_s + term_p + term_pv + term_f
    bound = rest + 2.0 ** -8 * (ya + rest)
    return torch.where(dead, zero, y), torch.where(dead, zero, bound)


def _gather(t, idx):
    """Rows idx of t (fp64); rows past the end read as zeros, as TMA fills them."""
    ok = idx < t.shape[0]
    g = t[idx.clamp(max=t.shape[0] - 1)].double()
    return torch.where(ok.reshape(-1, *([1] * (g.dim() - 1))), g, torch.zeros_like(g))


def _request_kv(k_nope, k_pe, v, kv0, n, h, mutation):
    """Keys [H, n, 192] and values [H, n, 128] the kernel (or a mutant) reads for one request."""
    dev = k_nope.device
    idx = kv0 + torch.arange(n, device=dev)
    kn = _gather(k_nope, idx).transpose(0, 1)  # [H, n, 128]
    vv = kn if mutation == "v_from_k_nope" else _gather(v, idx).transpose(0, 1)
    if mutation == "pe_per_head":  # k_pe addressed with the head as a row offset
        kp = torch.stack([_gather(k_pe, idx + hh) for hh in range(h)])
    else:
        kp = _gather(k_pe, idx)[None].expand(h, n, D_PE)
    if mutation == "pe_dropped":
        kp = torch.zeros_like(kp)
    if mutation == "head_swap":
        kn, vv = kn.flip(0), vv.flip(0)
    return torch.cat([kn, kp], 2), vv


def mla_prefill_exact(q, k_nope, k_pe, v, cu_seqlens_q, cu_seqlens_kv, scale, lossy=False,
                      mutation=None, rows=None):
    """q [Tq, H, 192], k_nope / v [Tkv, H, 128], k_pe [Tkv, 64] (any float dtype, one device);
    cu_seqlens_* int [B + 1]. Returns (y, B) float64 [Tq, H, 128] on q's device; with lossy=True
    (lossy oracle or mutant output, None). Rows of no request, and rows outside the bool mask
    `rows` [Tq], are NaN."""
    dev = q.device
    tq, h = q.shape[0], q.shape[1]
    y = torch.full((tq, h, DV), math.nan, dtype=torch.float64, device=dev)
    bnd = torch.full_like(y, math.nan)
    cq, ck = [int(x) for x in cu_seqlens_q], [int(x) for x in cu_seqlens_kv]
    sc = 1.0 / math.sqrt(DQK) if mutation == "scale_ignored" else scale
    for b in range(len(cq) - 1):
        s0, nq = cq[b], cq[b + 1] - cq[b]
        nk = ck[b + 1] - ck[b]
        if nq == 0:
            continue
        ri = torch.arange(nq, device=dev)
        if rows is not None:
            ri = ri[rows[s0:s0 + nq].to(dev)]
        if ri.numel() == 0:
            continue
        n_eff = nk
        if mutation == "next_request_visible":  # key count rounded up to whole tiles
            n_eff = (nk + TILE - 1) // TILE * TILE
        kv0 = cq[b] if mutation == "kv_offset_from_q" else ck[b]
        kr, vr = _request_kv(k_nope, k_pe, v, kv0, n_eff, h, mutation)
        pos = torch.arange(n_eff, device=dev)
        qb = q[s0:s0 + nq].double().transpose(0, 1)  # [H, nq, 192]
        step = max(1, _BUDGET // max(1, h * n_eff))
        for c0 in range(0, ri.numel(), step):
            rr = ri[c0:c0 + step]
            lim = n_eff - nq + rr
            if mutation == "top_left":
                lim = rr
            elif mutation == "causal_off_by_one":
                lim = lim + 1
            vis = (pos[None, :] <= lim[:, None]) & (pos[None, :] < n_eff)
            tile_hi = torch.clamp(nk - nq + (rr // TILE + 1) * TILE, 0, nk)
            n_tiles = ((tile_hi + TILE - 1) // TILE).double()
            yy, bb = _rows(qb[:, rr], kr, vr, vis, n_tiles, sc, lossy)
            y[s0 + rr] = yy.transpose(0, 1)
            if bb is not None:
                bnd[s0 + rr] = bb.transpose(0, 1)
    return (y, None) if lossy else (y, bnd)


def _args(d, device):
    return tuple(d[k].to(device) for k in ("q", "k_nope", "k_pe", "v")) + (
        d["cu_seqlens_q"], d["cu_seqlens_kv"], d["scale"])


def check(out, d, rows=None, device="cpu"):
    """Two-part check of a kernel (or mutant) output against synth.prefill_mla case `d`, on the
    query rows of the bool mask `rows` (default: all). The reference runs on `device`."""
    a = _args(d, device)
    exact, bound = mla_prefill_exact(*a, rows=rows)
    lossy, _ = mla_prefill_exact(*a, lossy=True, rows=rows)
    out = out.double().cpu()
    exact, bound, lossy = exact.cpu(), bound.cpu(), lossy.cpu()
    if rows is not None:
        out, exact, bound, lossy = out[rows], exact[rows], bound[rows], lossy[rows]
    return grade(out, exact, bound, lossy)


def mutant(d, mutation):
    """What a kernel with `mutation` would compute on case `d` (bf16 P, bf16 output)."""
    return mla_prefill_exact(*_args(d, "cpu"), lossy=True, mutation=mutation)[0]
