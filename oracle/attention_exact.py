"""ORACLE — test infrastructure only (see oracle/__init__.py).

Exact (fp64) FP8 attention on the dequantised inputs, with a per-element bound B on
|kernel - exact| derived from the kernels' own arithmetic, and the two-part check built on it.

Notation (one query row, natural-log units): s_j = q.k_j * cq * ck_j over the visible keys j,
m = max_j s_j, p_j = exp(s_j - m) (so max_j p_j = 1), L = sum_j p_j >= 1, y = vs * sum_j p_j v_j / L.
q, k, v are the e4m3 codes, cq = q_scale / sqrt(D) (times k_scale for per-tensor K), ck_j the
per-token k scale (1 for per-tensor K), vs the v scale.

What the kernels compute differently (csrc/decode_attn_fp8.cu, csrc/prefill_blocksparse_fp8.cu):

1. P rounding (dominant). P is stored as e4m3(256 * p~) with p~ = 2^(s - r) relative to a
   reference r <= m: the running maximum of a split-k chunk (decode, p~ <= 1) or the lazy maximum
   that lags the running one by up to 0.75 log2 (prefill, 256 p~ <= 430 < 448, never saturated).
   e4m3 rounding of a normal value is within 2^-4 of it; in the subnormal range the error is at
   most half the step 2^-9, i.e. 2^-10 in units of 256 p~, 2^-18 in units of p~. Converting to
   units of the true maximum multiplies by 2^(r - m) <= 1, so
       |dp_j| <= 2^-4 p_j + 2^-18,      term_P = vs * (2^-4 sum p_j |v_j| + 2^-18 sum |v_j|) / L.
   The row sum uses the unquantised values, so P rounding enters the numerator only.
2. Score and exponential error. Any relative error r_j of p_j that enters numerator and row sum
   alike moves y by sum_j p_j r_j (v_j - y) / sum_j p_j (1 + r_j), bounded with
   |v_j - y| <= |v_j| + |y| and the denominator >= L exp(-max delta). Per key,
       delta_j = FP8_ACC_EPS * QK_STEPS * sum_i |q_i k_ji| * |cq| ck_j      (fp8 wgmma accumulation)
               + 2^-22 (|s_j| + |m|)                                      (fp32 scale, subtract)
               + EXP_REL + n_tiles * 2^-21                                 (exponentials, rescales)
   and r_j <= expm1(delta_j). EXP_REL is the larger of ex2.approx's error and the error of the
   prefill's exp2_poly_pair polynomial (csrc/prefill_common.cuh), evaluated below in float32
   numpy over the polynomial's whole input range [-0.5, 0.5].
3. PV accumulation. Each m64nNk32 fp8 wgmma step adds rounding of at most FP8_ACC_EPS times the
   magnitude it accumulates (<= sum of |terms| of the chain). Decode starts a fresh chain per
   128-key tile (4 steps, then fp32); the prefill chains every visited tile of a Q tile
   (4 steps per tile): term_PV = vs * FP8_ACC_EPS * steps * sum_j (1 + 2^-4) p_j |v_j| / L.
4. Output rounding: bf16, relative 2^-8 of the kernel's value: 2^-8 (|y| + B_rest).
   fp32 epilogue / split-k combine arithmetic: 2^-20 vs sum_j p_j |v_j| / L.

FP8_ACC_EPS is the one constant not derived from the code. Hopper fp8 wgmma aligns the products
of a k = 32 step to the largest exponent and keeps about 14 significant bits (DESIGN §3.5; the
DeepSeek-V3 report measures ~2^-7 relative error at K = 4096, i.e. 128 steps). Two truncations
per step (the step's sum and its addition to the accumulator), each < 2^-13 of the chain's
magnitude, give FP8_ACC_EPS = 2^-12 per step.

The check has two parts (grade()):
  (a) |kernel - exact| <= B element-wise; cannot flake, since B is a worst case.
  (b) rel_l2(kernel - exact) <= AGG_C * rel_l2(lossy oracle - exact) + AGG_FLOOR. The kernel and
      the lossy oracle round the same P values with the same e4m3 grid, only against other maxima
      (chunk / lazy instead of the row maximum), so their rounding noise has the same size; AGG_C
      = 2 leaves room for that plus the fp8 accumulation noise the oracle does not have.
      AGG_FLOOR = 2^-8 covers outputs whose only error is the bf16 rounding (a dominant key with
      p = 1 is exact in e4m3).
"""
import math

import numpy as np
import torch

FP8_ACC_EPS = 2.0 ** -12
QK_STEPS = 4           # D = 128 as four k = 32 wgmma steps
PV_STEPS_PER_TILE = 4  # 128 keys per tile as four k = 32 steps
TILE = 128
AGG_C = 2.0
AGG_FLOOR = 2.0 ** -8


def exp2_poly_rel_err(n=1 << 20):
    """Max relative error of exp2_poly_pair's polynomial on [-0.5, 0.5], evaluated in float32
    with the kernel's coefficients and Horner order."""
    f = np.linspace(-0.5, 0.5, n, dtype=np.float32)
    c3, c2, c1, c0 = (np.float32(v) for v in (0.0551716685, 0.2426111251, 0.6932609677,
                                              0.9999280572))
    q = (f * c3 + c2).astype(np.float32)
    q = (q * f + c1).astype(np.float32)
    q = (q * f + c0).astype(np.float32)
    ref = np.exp2(f.astype(np.float64))
    return float(np.max(np.abs(q.astype(np.float64) - ref) / ref))


# ex2.approx.f32: relative error below 2^-22 (PTX ISA); the polynomial is far worse. The extra
# 2^-21 covers the float32 rounding of the FMAs that numpy does as separate operations.
EXP_REL = max(exp2_poly_rel_err(), 2.0 ** -22) + 2.0 ** -21


def _rows(qc, kc, vc, cq, ck, vis, vs, pv_steps, n_tiles):
    """One (request, kv head) problem in fp64. qc [R, D], kc/vc [N, D] codes; cq [R]; ck [N];
    vis [R, N] bool; vs scalar; pv_steps, n_tiles [R]. Returns y, B [R, D] (NaN rows where a row
    sees no key)."""
    raw = qc @ kc.T
    absraw = qc.abs() @ kc.abs().T
    s = raw * cq[:, None] * ck[None, :]
    s = torch.where(vis, s, torch.full_like(s, -math.inf))
    m = s.max(dim=1, keepdim=True).values
    dead = ~torch.isfinite(m)
    m = torch.where(dead, torch.zeros_like(m), m)
    p = torch.exp(s - m)  # 0 on masked keys
    L = p.sum(1, keepdim=True)
    va = vc.abs()
    y = (p @ vc) / L
    ya = y.abs()
    visf = vis.to(p.dtype)

    delta = (FP8_ACC_EPS * QK_STEPS * absraw * cq.abs()[:, None] * ck[None, :]
             + 2.0 ** -22 * (s.abs() + m.abs()) + EXP_REL + n_tiles[:, None] * 2.0 ** -21)
    delta = torch.where(vis, delta, torch.zeros_like(delta))
    r = torch.expm1(delta)
    lmin = L * torch.exp(-delta.max(dim=1, keepdim=True).values)
    pr = p * r
    phi = p + pr
    term_s = (pr @ va + ya * pr.sum(1, keepdim=True)) / lmin
    term_p = (2.0 ** -4 * (phi @ va) + 2.0 ** -18 * (visf @ va)) / lmin
    term_pv = FP8_ACC_EPS * pv_steps[:, None] * ((1 + 2.0 ** -4) * (phi @ va)
                                                 + 2.0 ** -18 * (visf @ va)) / lmin
    term_f = 2.0 ** -20 * (phi @ va) / lmin
    rest = abs(vs) * (term_s + term_p + term_pv + term_f)
    y = y * vs
    bound = rest + 2.0 ** -8 * (y.abs() + rest)
    nan = torch.full_like(y, math.nan)
    return torch.where(dead, nan, y), torch.where(dead, nan, bound)


def _paged(cache, ids, n, head):
    return cache[ids.long()].reshape(-1, cache.shape[2], cache.shape[3])[:n, head].double()


def _kpt_scales(kscale, ids, n, head):
    ks = kscale.contiguous()
    if ks.element_size() == 1:
        ks = ks.view(torch.float32)
    # [blocks, bs/32, Hkv, 32]: token t of a page -> [page, t // 32, head, t % 32]
    return ks[ids.long()][:, :, head].reshape(-1)[:n].double()


def decode_fp8_exact(q, kcache, vcache, block_ids, kv_lens_total, q_scale, k_scale, v_scale,
                     num_seq_q, k_per_token=False):
    """Exact paged decode attention and its bound, arguments as oracle.attention.decode_fp8_*
    (k_per_token selects decode_fp8_kpertoken's scales). Returns (y, B), float64 [B*Sq, Hq, D]."""
    nb = kv_lens_total.shape[0]
    hq, d = q.shape[1], q.shape[2]
    hkv, bs = kcache.shape[2], kcache.shape[1]
    g = hq // hkv
    qv = q.reshape(nb, num_seq_q, hq, d).double()
    qs = q_scale.reshape(nb, num_seq_q, hq).double()
    y = torch.empty(nb, num_seq_q, hq, d, dtype=torch.float64)
    bound = torch.empty_like(y)
    for bi in range(nb):
        n = int(kv_lens_total[bi])
        ids = block_ids[bi, :(n + bs - 1) // bs]
        pos = torch.arange(n)
        lim = n - num_seq_q + torch.arange(num_seq_q)  # last visible key of each MTP row
        for h in range(hkv):
            kc, vc = _paged(kcache, ids, n, h), _paged(vcache, ids, n, h)
            if k_per_token:
                ck, vs = _kpt_scales(k_scale, ids, n, h), float(v_scale[h])
                kt = 1.0
            else:
                ck, vs, kt = torch.ones(n, dtype=torch.float64), float(v_scale[0]), float(k_scale[0])
            # rows ordered (q head in group, MTP row)
            qc = qv[bi, :, h * g:(h + 1) * g].transpose(0, 1).reshape(-1, d)
            cq = qs[bi, :, h * g:(h + 1) * g].transpose(0, 1).reshape(-1) * kt / math.sqrt(d)
            vis = (pos[None, :] <= lim[:, None]).repeat(g, 1)
            rows = qc.shape[0]
            steps = torch.full((rows,), float(PV_STEPS_PER_TILE), dtype=torch.float64)
            tiles = torch.full((rows,), float((n + TILE - 1) // TILE), dtype=torch.float64)
            yr, br = _rows(qc, kc, vc, cq, ck, vis, vs, steps, tiles)
            y[bi, :, h * g:(h + 1) * g] = yr.reshape(g, num_seq_q, d).transpose(0, 1)
            bound[bi, :, h * g:(h + 1) * g] = br.reshape(g, num_seq_q, d).transpose(0, 1)
    return y.reshape(-1, hq, d), bound.reshape(-1, hq, d)


def prefill_visible(nq, nkv, block_mask_b=None):
    """[Hq or 1, nq, nkv] bool: causal limit (row i sees keys <= nkv - nq + i) and the block mask,
    where KV tiles past the mask's width are skipped except the first one (oracle/prefill.py)."""
    cm = torch.tril(torch.ones(nkv, nkv, dtype=torch.bool))[nkv - nq:, :].unsqueeze(0)
    if block_mask_b is None:
        return cm
    em = block_mask_b.bool().repeat_interleave(TILE, -2)[:, :nq].repeat_interleave(TILE, -1)
    if em.shape[-1] < nkv:
        pad = torch.zeros(em.shape[0], nq, nkv - em.shape[-1], dtype=torch.bool)
        pad[:, :, :TILE] = True
        em = torch.cat([em, pad], -1)
    return em[:, :, :nkv] & cm


def prefill_fp8_exact(q, kcache, vcache, qscale, kscale, vscale, cu_seqlens_q, seqlens_kv,
                      block_ids, block_mask=None, k_per_token=False):
    """Exact block-sparse / dense prefill and its bound, arguments as
    oracle.prefill.blocksparse_prefill. Returns (y, B), float64 [total, Hq, D]; rows that see no
    key are NaN in both."""
    total, hq, d = q.shape
    bs, hkv = kcache.shape[1], kcache.shape[2]
    g = hq // hkv
    y = torch.full((total, hq, d), math.nan, dtype=torch.float64)
    bound = torch.full_like(y, math.nan)
    for i in range(seqlens_kv.shape[0]):
        s0, s1 = int(cu_seqlens_q[i]), int(cu_seqlens_q[i + 1])
        nq, nkv = s1 - s0, int(seqlens_kv[i])
        if nq == 0:
            continue
        ids = block_ids[i, :(nkv + bs - 1) // bs]
        vis_all = prefill_visible(nq, nkv, None if block_mask is None else block_mask[i])
        # fp8 wgmma chains O over every visited tile of the row's Q tile (its last row's extent)
        tile_end = torch.clamp((torch.arange(nq) // TILE + 1) * TILE, max=nq) - 1
        ntile = ((nkv - nq + tile_end + TILE) // TILE).clamp_min(0).double()
        for h in range(hkv):
            kc, vc = _paged(kcache, ids, nkv, h), _paged(vcache, ids, nkv, h)
            if k_per_token:
                ck, vs, kt = _kpt_scales(kscale, ids, nkv, h), float(vscale[h]), 1.0
            else:
                ck, vs, kt = torch.ones(nkv, dtype=torch.float64), float(vscale[0]), float(kscale[0])
            for hh in range(h * g, (h + 1) * g):
                qc = q[s0:s1, hh].double()
                cq = qscale[i, hh, :nq].double() * kt / math.sqrt(d)
                vis = vis_all[hh if vis_all.shape[0] > 1 else 0]
                yr, br = _rows(qc, kc, vc, cq, ck, vis, vs, PV_STEPS_PER_TILE * ntile, ntile)
                y[s0:s1, hh], bound[s0:s1, hh] = yr, br
    return y, bound


def _rel(a, ref):
    return float((a - ref).norm() / ref.norm().clamp_min(1e-30))


def grade(out, exact, bound, lossy):
    """Both checks. out / lossy: kernel and lossy-oracle outputs; exact, bound from *_exact.
    Returns a dict with ok_a, ok_b, the worst err/B, and the two relative L2 errors."""
    out, lossy = out.double().cpu(), lossy.double().cpu()
    nan = torch.isnan(exact)
    nan_ok = bool(torch.equal(torch.isnan(out), nan))
    keep = ~nan
    o, e, b, l = out[keep], exact[keep], bound[keep], lossy[keep]
    finite = bool(torch.isfinite(o).all())
    err = (o - e).abs()
    ratio = (float(torch.where(err == 0, torch.zeros_like(err), err / b).max())
             if o.numel() and finite else math.inf)
    rel_k, rel_o = (_rel(o, e), _rel(l, e)) if finite else (math.inf, _rel(l, e))
    ok_a = nan_ok and finite and ratio <= 1.0
    ok_b = finite and rel_k <= AGG_C * rel_o + AGG_FLOOR
    return dict(ok_a=ok_a, ok_b=ok_b, worst=ratio, rel=rel_k, rel_oracle=rel_o, nan_ok=nan_ok)


def assert_exact(out, exact, bound, lossy, tag=""):
    r = grade(out, exact, bound, lossy)
    assert r["nan_ok"], f"{tag}: NaN rows differ from the exact reference"
    assert r["ok_a"], f"{tag}: |out - exact| / B = {r['worst']:.3f} > 1"
    assert r["ok_b"], (f"{tag}: rel L2 {r['rel']:.4g} > {AGG_C} * {r['rel_oracle']:.4g} "
                       f"+ {AGG_FLOOR:.4g}")
    return r
