"""Oracle of the Stem block-mask stages (hpc/stem.py), one function per stage.

The prep stages and the GEMM compute in float64 and return, per element, the bound that the
kernel's bf16 / fp32 rounding allows; the TPD stage is exact: integer keys and the budget in fp32
with every operation rounded as the kernel rounds it (the decay as one fused multiply-add).
Each stage takes the kernel's own inputs to that stage, so a stage is checked on its own."""
import math
from fractions import Fraction

import numpy as np
import torch

BLOCK = 128
STRIDE = 16
SAMPLES = BLOCK // STRIDE
U = 2.0 ** -24  # fp32 unit roundoff


def cdiv(a, b):
    return -(-a // b)


def c_div(a, b):
    """C integer division (truncates toward zero)."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def causal_offset(q_len, kv_len):
    return c_div(kv_len - q_len + BLOCK - 1, BLOCK)


def half_ulp_bf16(y):
    """Half a bf16 ulp at |y| (float64 array): the rounding error of fp32 -> bf16."""
    a = np.abs(np.asarray(y, dtype=np.float64))
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -126)))
    return 2.0 ** (e - 8)


def _pages(cache, ids, n, head):
    """[n, 128] float64 rows of one head of a paged cache [blocks, page, Hkv, 128]."""
    page = cache.shape[1]
    rows = cache[ids[:cdiv(n, page)].long()].float().double()  # [np, page, Hkv, 128]
    return rows.reshape(-1, cache.shape[2], cache.shape[3])[:n, head].numpy()


def _token_kscale(kscale, ids, n, head, page):
    """Per-token K scales [n] of one head: kscale[page, (row % page) / 32, head, row % 32]."""
    ks = kscale.view(torch.float32) if kscale.dtype != torch.float32 else kscale
    per = ks[ids[:cdiv(n, page)].long(), :, head, :].reshape(-1)  # [np * page]
    return per[:n].double().numpy()


def _group_sums(rows, scale, n_blocks):
    """Group sums of rows [n, 128] times per-row scale [n]: ([Kb, 16, 128] value, sum |term|)."""
    n = rows.shape[0]
    pad = n_blocks * BLOCK - n
    terms = np.concatenate([rows * scale[:, None], np.zeros((pad, rows.shape[1]))])
    terms = terms.reshape(n_blocks, SAMPLES, STRIDE, rows.shape[1])  # row = kb*128 + r*16 + g
    return terms.sum(1), np.abs(terms).sum(1)


def flat_bound(y, abs_sum, exact_sum):
    """Bound of a kernel group sum rounded to bf16: half an ulp plus the fp32 accumulation."""
    d = np.zeros_like(y) if exact_sum else SAMPLES * 2 * U * abs_sum + U * np.abs(y)
    return half_ulp_bf16(np.abs(y) + d) + d


def kv_prep(kcache, vcache, kscale, vscale, kv_indices, kv_seq_lens, lambda_mag=0.3, quant_type=1):
    """Returns per request b a dict: kflat [Hkv, Kb, 2048], kflat_bound, kflat_abs (sum of the
    |terms| of each group sum), vbias [Hkv, Kb], vbias_bound (float64), for the request's own Kb = ceil(kv_len / 128) blocks."""
    page, hkv = kcache.shape[1], kcache.shape[2]
    out = []
    for b in range(kv_seq_lens.shape[0]):
        n = int(kv_seq_lens[b])
        nkb = cdiv(n, BLOCK)
        ids = kv_indices[b]
        kf = np.zeros((hkv, nkb, STRIDE * 128))
        kfb = np.zeros_like(kf)
        kfa = np.zeros_like(kf)  # sum of |terms| of each group sum
        vb = np.zeros((hkv, nkb))
        vbb = np.zeros_like(vb)
        for h in range(hkv if nkb else 0):
            k = _pages(kcache, ids, n, h)
            v = _pages(vcache, ids, n, h)
            if quant_type == 1:
                s, ab = _group_sums(k, np.ones(n), nkb)
                s, ab = s * float(kscale[0]), ab * abs(float(kscale[0]))
                vs = float(vscale[0])
            else:
                s, ab = _group_sums(k, _token_kscale(kscale, ids, n, h, page), nkb)
                vs = float(vscale[h])
            bnd = flat_bound(s, ab, quant_type == 1)
            kf[h] = s[:, ::-1, :].reshape(nkb, -1)  # group g -> segment 15 - g
            kfb[h] = bnd[:, ::-1, :].reshape(nkb, -1)
            kfa[h] = ab[:, ::-1, :].reshape(nkb, -1)
            vb[h], vbb[h] = vbias_stats(v, vs, nkb, lambda_mag)
        out.append(dict(kflat=kf, kflat_bound=kfb, kflat_abs=kfa, vbias=vb, vbias_bound=vbb))
    return out


def vbias_stats(v, vs, nkb, lambda_mag, ddof=1, pad_rows=True):
    """vbias of one (request, head) from its V rows [n, 128] and the bound of the kernel's fp32
    arithmetic. ddof / pad_rows exist to express simulated bugs in the tests."""
    n = v.shape[0]
    norms = np.sqrt(((v * vs) ** 2).sum(1))
    full = np.zeros(nkb * BLOCK)
    full[:n] = norms
    x = full.reshape(-1, STRIDE).max(1)  # [nkb * 8]
    if not pad_rows:
        x = x[:cdiv(n, STRIDE)]
    m_n = x.shape[0]
    lg = np.log(x + 1e-6)
    mean = lg.mean()
    sd = math.sqrt(((lg - mean) ** 2).sum() / (m_n - ddof)) if m_n > ddof else 0.0
    inv = 1.0 / (sd + 1e-6)
    z = (lg - mean) * inv
    if not pad_rows:
        z = np.concatenate([z, np.full(nkb * SAMPLES - m_n, -np.inf)])
    vb = (lambda_mag * np.maximum(z, 0.0)).reshape(nkb, SAMPLES).mean(1)
    # error propagation of the kernel's fp32 path (norm, logf, block sums, std, scaling)
    e_l = 40 * U * x / (x + 1e-6) + 2 * U * np.abs(lg) + U
    if not pad_rows:
        e_l = np.concatenate([e_l, np.zeros(nkb * SAMPLES - m_n)])
        lg = np.concatenate([lg, np.zeros(nkb * SAMPLES - m_n)])
    k_acc = m_n / 256 + 16
    e_m = (e_l.sum() + k_acc * U * np.abs(lg).sum()) / m_n + U * abs(mean)
    d = np.abs(lg - mean)
    e_d = e_l + e_m + U * d
    var = (d ** 2).sum()
    e_var = (2 * d * e_d + e_d ** 2).sum() + (k_acc + 2) * U * var
    e_s = 0.5 * e_var / max(var, 1e-300) * sd + 4 * U * sd
    e_inv = inv * (e_s / (sd + 1e-6) + 2 * U)
    zz = np.abs(np.where(np.isfinite(z), z, 0.0))
    e_z = e_d * inv + d * e_inv + U * zz
    e_z = np.where(np.isfinite(z) & (z > -e_z), e_z, 0.0)
    e_v = lambda_mag * e_z.reshape(nkb, SAMPLES).mean(1) + 12 * U * np.abs(vb)
    return vb, e_v


def q_prep(q, qscale, q_seq_lens, cu_seqlens_q):
    """Per request b: dict qflat [Hq, Qb, 2048], qflat_bound (float64), Qb = ceil(q_len / 128)."""
    hq = q.shape[1]
    out = []
    for b in range(q_seq_lens.shape[0]):
        n = int(q_seq_lens[b])
        s0 = int(cu_seqlens_q[b])
        nqb = cdiv(n, BLOCK)
        qf = np.zeros((hq, nqb, STRIDE * 128))
        qfb = np.zeros_like(qf)
        for h in range(hq if nqb else 0):
            rows = q[s0:s0 + n, h].float().double().numpy()
            s, ab = _group_sums(rows, qscale[b, h, :n].double().numpy(), nqb)
            qf[h] = s.reshape(nqb, -1)
            qfb[h] = flat_bound(s, ab, False).reshape(nqb, -1)
        out.append(dict(qflat=qf, qflat_bound=qfb))
    return out


def neg_inf_mask(q_len, kv_len, max_qb, max_kb, causal=True, offset=None):
    """[max_qb, max_kb] bool: where the logits are -inf."""
    nqb, nkb = cdiv(q_len, BLOCK), cdiv(kv_len, BLOCK)
    off = causal_offset(q_len, kv_len) if offset is None else offset
    qb = np.arange(max_qb)[:, None]
    kb = np.arange(max_kb)[None, :]
    dead = (qb >= nqb) | (kb >= nkb)
    if causal:
        dead = dead | (qb + off < kb)
    return dead


def gemm(qflat, kflat, vbias, q_seq_lens, kv_seq_lens, causal=True):
    """From the kernel's own qflat [B, Hq, Qb, 2048] bf16, kflat [B, Hkv, Kb, 2048] bf16 and vbias
    [B, Hkv, Kb] fp32: (logits, bound, dead), float64 [B, Hq, Qb, Kb] / bool. Elements where dead
    is set must be -inf exactly; elsewhere |kernel - logits| <= bound."""
    q = qflat.double().numpy()
    k = kflat.double().numpy()
    vb = np.nan_to_num(vbias.double().numpy())  # blocks past a request are never written
    B, hq, max_qb, _ = q.shape
    hkv, max_kb = k.shape[1], k.shape[2]
    g = hq // hkv
    y = np.zeros((B, hq, max_qb, max_kb))
    bound = np.zeros_like(y)
    dead = np.zeros(y.shape, dtype=bool)
    for b in range(B):
        dm = neg_inf_mask(int(q_seq_lens[b]), int(kv_seq_lens[b]), max_qb, max_kb, causal)
        for h in range(hq):
            qq = np.where(dm.all(1)[:, None], 0.0, q[b, h])  # rows never used may hold garbage
            kk = np.where(dm.all(0)[:, None], 0.0, k[b, h // g])
            kk = np.nan_to_num(kk)
            qq = np.nan_to_num(qq)
            acc = qq @ kk.T / 64.0
            mag = np.abs(qq) @ np.abs(kk).T / 64.0
            val = acc + vb[b, h // g][None, :]
            d = 2048 * 2.0 ** -23 * mag + U * np.abs(val)
            y[b, h] = np.where(dm, -np.inf, val)
            bound[b, h] = np.where(dm, 0.0, half_ulp_bf16(np.abs(val) + d) + d)
            dead[b, h] = dm
    return y, bound, dead


# ---------------------------------------------------------------------------------------------
# TPD (exact)
# ---------------------------------------------------------------------------------------------
NON_FINITE = 0x007F


def ordered_keys(bits):
    """bf16 bit patterns (uint16 array) -> ordered 16-bit keys; non-finite (+-inf, NaN) -> 0x007F."""
    bits = np.asarray(bits, dtype=np.uint16).astype(np.int64)
    key = np.where(bits & 0x8000, (~bits) & 0xFFFF, bits ^ 0x8000)
    return np.where((bits & 0x7F80) == 0x7F80, NON_FINITE, key)


def _round_f32(v: Fraction) -> np.float32:
    """The fp32 nearest to the rational v, ties to even (one rounding)."""
    f = np.float32(float(v))
    best = None
    for c in (np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))):
        if not np.isfinite(c):
            continue
        err = abs(Fraction(float(c)) - v)
        even = (int(np.array(c, dtype=np.float32).view(np.uint32)) & 1) == 0
        key = (err, not even)
        if best is None or key < best[0]:
            best = (key, c)
    return best[1]


def budget(q_pos, prompt_blocks, alpha=1.0, rate_m=0.2, bias_m=30, rate_l=0.1, bias_l=30,
           fma=True):
    """Top-k budget of absolute query block q_pos, in fp32 as the kernel computes it.
    fma=False rounds the product of the decay separately (a simulated bug)."""
    f32 = np.float32
    P = int(prompt_blocks)
    if P < 56:
        k = P
    elif P < 160:
        k = int(f32(P) * f32(rate_m)) + int(bias_m)
    else:
        k = int(f32(P) * f32(rate_l)) + int(bias_l)
    decay = P - k
    if q_pos < k or decay <= 1:
        return k
    kf = f32(k)
    k_end = kf * f32(alpha)
    t = f32(q_pos - k) / f32(decay - 1)
    diff = k_end - kf
    if fma:
        v = _round_f32(Fraction(float(t)) * Fraction(float(diff)) + Fraction(float(kf)))
    else:
        v = f32(t * diff) + kf
    bud = int(math.floor(float(v)))
    return max(1, min(bud, k))


def threshold(keys, bud):
    """Largest T with count(keys >= T) >= bud over the finite keys (every finite key when the
    budget covers them all; none when bud <= 0)."""
    fin = np.sort(keys[keys != NON_FINITE])[::-1]
    if bud <= 0:
        return 0xFFFF
    if bud >= fin.shape[0]:
        return NON_FINITE + 1
    return int(fin[bud - 1])


def tpd(block_logits, q_seq_lens, kv_seq_lens, num_prompt_tokens, alpha=1.0, initial_blocks=4,
        window_size=4, rate_m=0.2, bias_m=30, rate_l=0.1, bias_l=30, budget_fn=None):
    """Exact mask u8 [B, H, Qb, Kb] from bf16 block_logits (torch, any device)."""
    bits = block_logits.contiguous().cpu().view(torch.int16).numpy().astype(np.uint16)
    B, H, max_qb, max_kb = bits.shape
    mask = np.zeros(bits.shape, dtype=np.uint8)
    bf = budget if budget_fn is None else budget_fn
    for b in range(B):
        ql, kl = int(q_seq_lens[b]), int(kv_seq_lens[b])
        qi, ki = cdiv(ql, BLOCK), min(cdiv(kl, BLOCK), max_kb)
        if qi == 0 or ki == 0:
            continue
        P = cdiv(int(num_prompt_tokens[b]), BLOCK)
        off = causal_offset(ql, kl)
        cols = np.arange(ki)
        for qr in range(min(qi, max_qb)):
            bud = bf(qr + off, P, alpha, rate_m, bias_m, rate_l, bias_l)
            diag = min(qr + off, ki - 1)
            fixed = ((cols < initial_blocks) | ((cols <= diag) & (cols > diag - window_size))
                     | (cols == diag))
            for h in range(H):
                keys = ordered_keys(bits[b, h, qr, :ki])
                T = threshold(keys, bud)
                mask[b, h, qr, :ki] = ((keys >= T) & (keys != NON_FINITE) | fixed).astype(np.uint8)
    return mask
