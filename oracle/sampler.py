"""numpy restatement of the fused sampler (hpc/sampler.py), fp32 arithmetic made explicit.

`fused_sampler` and `temperature_sample` follow DESIGN.md §3.10 step by step. `mutations` names
deliberate faults (see MUTATIONS); tests use them to show that their inputs tell a correct sampler
from a wrong one. `philox4x32_10` and `philox_gumbel` restate the kernel's internal noise.
"""
import numpy as np

F32 = np.float32
NEG_INF = F32(-np.inf)

MUTATIONS = (
    "topp_inclusive",    # top-p on the inclusive cumulative sum
    "topp_ignored",      # top-p never drops a candidate
    "tie_larger_id",     # ties go to the larger token id (selection and argmax)
    "k_off_by_one",      # K_b = topk_b + 1 for topk_b in range
    "softmax_over_max",  # AFTER_TOPK softmax over max_topk candidates instead of K_b
    "noise_by_rank",     # noise g[b, rank] instead of g[b, token]
    "penalty_sign",      # positive logits multiplied by rp, the rest divided
    "mask_bit_msb",      # bit 7 - v % 8 instead of v % 8
    "mask_row_b",        # penalty_mask row b instead of slot_id[b]
    "temperature_ignored",
    "draft_ignored",
    "stride_ignored",    # rows read as if stride(0) == V
)

# ---------------------------------------------------------------------------------------------------
# Philox4x32-10 (Salmon, Moraes, Dror, Shaw, SC'11), as Random123 defines it
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
_MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr uint32 [..., 4], key uint32 [..., 2] (broadcast) -> uint32 [..., 4]."""
    c = [np.asarray(ctr, np.uint32)[..., i].astype(np.uint64) for i in range(4)]
    k0 = np.asarray(key, np.uint32)[..., 0].copy()
    k1 = np.asarray(key, np.uint32)[..., 1].copy()
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = _M0 * c[0]
            p1 = _M1 * c[2]
            hi0, lo0 = p0 >> np.uint64(32), p0 & _MASK32
            hi1, lo1 = p1 >> np.uint64(32), p1 & _MASK32
            c = [hi1 ^ c[1] ^ k0.astype(np.uint64), lo1, hi0 ^ c[3] ^ k1.astype(np.uint64), lo0]
            k0 = (k0 + _W0).astype(np.uint32)
            k1 = (k1 + _W1).astype(np.uint32)
    return np.stack([x.astype(np.uint32) for x in c], axis=-1)


def uniform_from_bits(x):
    """The top 23 bits of x -> u = (x >> 9) * 2^-23 + 2^-24 in [2^-24, 1 - 2^-24], exact in fp32."""
    x = np.asarray(x, np.uint32)
    return ((x >> np.uint32(9)).astype(F32) * F32(2.0 ** -23) + F32(2.0 ** -24)).astype(F32)


def gumbel_from_uniform(u):
    with np.errstate(divide="ignore"):
        return (-np.log(-np.log(u.astype(F32)))).astype(F32)


def philox_gumbel(seed: int, offset: int, batch: int, vocab: int):
    """The kernel's noise [batch, vocab]: counter (v // 4, row, offset lo, offset hi), key = seed,
    output word v % 4."""
    q = np.arange(vocab // 4, dtype=np.uint32)
    ctr = np.zeros((batch, vocab // 4, 4), np.uint32)
    ctr[..., 0] = q[None, :]
    ctr[..., 1] = np.arange(batch, dtype=np.uint32)[:, None]
    ctr[..., 2] = np.uint32(offset & 0xFFFFFFFF)
    ctr[..., 3] = np.uint32(offset >> 32)
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], np.uint32)
    bits = philox4x32_10(ctr, key).reshape(batch, vocab)
    return gumbel_from_uniform(uniform_from_bits(bits))


# ---------------------------------------------------------------------------------------------------
def _rows(storage, vocab, mutations):
    """[B, V] fp32 view of the logits rows held in `storage` [B, row_stride]."""
    storage = np.asarray(storage)
    B = storage.shape[0]
    if "stride_ignored" in mutations:
        flat = storage.reshape(-1)
        rows = np.stack([flat[b * vocab:(b + 1) * vocab] for b in range(B)]) if B else storage[:, :vocab]
    else:
        rows = storage[:, :vocab]
    return rows.astype(F32)


def _per_row(v, B, dtype):
    a = np.asarray(v)
    return np.broadcast_to(a.astype(dtype), (B,)).copy() if a.ndim == 0 else a.astype(dtype).copy()


def _penalise_and_temper(x, mask, slot, rp, temp, mutations):
    B, V = x.shape
    x = x.copy()
    v = np.arange(V)
    for b in range(B):
        if mask is not None and rp[b] > 0:
            row = b if "mask_row_b" in mutations else int(slot[b])
            bit = (7 - v % 8) if "mask_bit_msb" in mutations else v % 8
            hit = ((mask[row, v // 8] >> bit) & 1).astype(bool)
            r = F32(rp[b])
            inv = F32(1.0) / r
            pos = x[b] > 0
            if "penalty_sign" in mutations:
                x[b] = np.where(hit, np.where(pos, x[b] * r, x[b] * inv), x[b])
            else:
                x[b] = np.where(hit, np.where(pos, x[b] * inv, x[b] * r), x[b])
        if temp[b] > 0 and "temperature_ignored" not in mutations:
            x[b] = x[b] / F32(temp[b])
    return x


def top_candidates(xr, k, larger_id_first=False):
    """Token ids of the k largest values of row xr, by value descending then id ascending."""
    V = xr.shape[0]
    idx = np.argpartition(-xr, k - 1)[:k] if k < V else np.arange(V)
    thr = xr[idx].min()
    gt = np.nonzero(xr > thr)[0]
    eq = np.nonzero(xr == thr)[0]
    eq = eq[::-1] if larger_id_first else eq
    cand = np.concatenate([gt, eq[:k - gt.size]])
    ids = -cand if larger_id_first else cand
    return cand[np.lexsort((ids, -xr[cand].astype(np.float64)))]


def _argmax_smallest_id(key, tok, larger=False):
    best = key.max()
    ties = tok[key == best]
    return int(ties.max() if larger else ties.min())


def fused_sampler(storage, vocab, *, penalty_mask=None, slot_id=None, repetition_penalty=0.0,
                  temperature=0.0, softmax_policy=0, topk=0, topp=0.0, max_topk=32, noise,
                  mutations=(), detail=False):
    """Full path. Returns (tokens int32 [B], updated penalty mask or None[, per-row details])."""
    x0 = _rows(storage, vocab, mutations)
    B, V = x0.shape
    rp = _per_row(repetition_penalty, B, np.float32)
    temp = _per_row(temperature, B, np.float32)
    tk = _per_row(topk, B, np.int64)
    tp = _per_row(topp, B, np.float32)
    mask = None if penalty_mask is None else np.array(penalty_mask, np.uint8)
    x = _penalise_and_temper(x0, mask, slot_id, rp, temp, mutations)
    tie_big = "tie_larger_id" in mutations
    out = np.zeros(B, np.int32)
    details = []
    for b in range(B):
        xr = x[b]
        cand = top_candidates(xr, max_topk, tie_big)
        kb = int(tk[b]) if 1 <= tk[b] <= max_topk else max_topk
        if "k_off_by_one" in mutations and 1 <= tk[b] <= max_topk:
            kb = min(kb + 1, max_topk)
        ksm = max_topk if "softmax_over_max" in mutations else kb
        xc = xr[cand]
        p = np.zeros(max_topk, F32)
        with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
            if softmax_policy == 1:
                M = xr.max()
                e_all = np.where(xr == NEG_INF, F32(0), np.exp(xr - M)).astype(F32)
                S = F32(e_all.astype(np.float64).sum())
                e = np.where(xc == NEG_INF, F32(0), np.exp(xc - M)).astype(F32)
                e[kb:] = 0
                p = np.where(e > 0, e / S, F32(0)).astype(F32)
            elif softmax_policy == 2:
                M = xc[0]
                e = np.where(xc == NEG_INF, F32(0), np.exp(xc - M)).astype(F32)
                e[ksm:] = 0
                S = F32(e.astype(np.float64).sum())
                p = np.where(e > 0, e / S, F32(0)).astype(F32)
                p[kb:] = 0
            val = xc if softmax_policy == 0 else np.where(p > 0, np.log(p), NEG_INF).astype(F32)
        keep = np.arange(max_topk) < kb
        excl = (np.cumsum(p, dtype=np.float64) - p).astype(F32)
        if tp[b] > 0 and "topp_ignored" not in mutations:
            s = (excl + p).astype(F32) if "topp_inclusive" in mutations else excl
            keep &= (np.arange(max_topk) == 0) | (s < tp[b])
        g = noise[b, np.arange(max_topk)] if "noise_by_rank" in mutations else noise[b, cand]
        key = np.where(keep, (val + g).astype(F32), NEG_INF).astype(F32)
        tok = _argmax_smallest_id(key[:kb], cand[:kb], tie_big)
        out[b] = tok
        if mask is not None:
            row = b if "mask_row_b" in mutations else int(slot_id[b])
            bit = (7 - tok % 8) if "mask_bit_msb" in mutations else tok % 8
            mask[row, tok // 8] |= np.uint8(1 << bit)
        if detail:
            details.append(dict(cand=cand[:kb], x=xc[:kb].astype(np.float64), p_excl=excl[:kb], kb=kb,
                                topp=float(tp[b]), policy=softmax_policy, g=noise[b, cand[:kb]],
                                keep=keep[:kb], xr=xr))
    return (out, mask, details) if detail else (out, mask)


def temperature_sample(storage, vocab, *, temperature, noise, draft_token_ids=None, mutations=()):
    """Fast path: argmax of x / t + g (ties to the smaller id), draft token excluded; rows with
    t <= 0 (or NaN) take the argmax of the logits."""
    x = _rows(storage, vocab, mutations)
    B, V = x.shape
    temp = _per_row(temperature, B, np.float32)
    out = np.zeros(B, np.int32)
    for b in range(B):
        s = x[b].copy()
        if temp[b] > 0:
            t = F32(1) if "temperature_ignored" in mutations else F32(temp[b])
            s = ((s / t).astype(F32) + noise[b]).astype(F32)
        if draft_token_ids is not None and "draft_ignored" not in mutations:
            d = int(draft_token_ids[b])
            if 0 <= d < V:
                s[d] = NEG_INF
        best = s.max()
        ties = np.nonzero(s == best)[0]
        out[b] = ties.max() if "tie_larger_id" in mutations else ties.min()
    return out


# ---------------------------------------------------------------------------------------------------
def row_margins(d, noise_row=None):
    """fp64 margins of one full-path row from `fused_sampler(..., detail=True)` details:
    (top-p margin, key gap). The top-p margin is the distance of the exclusive cumulative sum from
    topp at every rank whose keep/drop decision would change the token; the key gap is the distance
    from the winning key to the runner-up. inf where an exact rule decides (no top-p, no finite
    runner-up, or a row of -inf keys)."""
    x = d["x"]
    kb = d["kb"]
    g = d["g"].astype(np.float64)
    if d["policy"] == 0:
        val = x.copy()
    else:
        if d["policy"] == 1:
            xr = d["xr"].astype(np.float64)
            xr = xr[np.isfinite(xr)]
            lse = xr.max() + np.log(np.exp(xr - xr.max()).sum()) if xr.size else -np.inf
        else:
            xf = x[np.isfinite(x)]
            lse = xf.max() + np.log(np.exp(xf - xf.max()).sum()) if xf.size else -np.inf
        with np.errstate(invalid="ignore"):
            val = np.where(np.isfinite(x), x - lse, -np.inf)
    p = np.where(np.isfinite(val), np.exp(val), 0.0) if d["policy"] else np.zeros(kb)
    excl = np.cumsum(p) - p

    def winner(keep):
        with np.errstate(invalid="ignore"):
            key = np.where(keep, val + g, -np.inf)
        if not np.isfinite(key).any():
            return int(d["cand"].min()), np.inf
        order = np.argsort(-key, kind="stable")
        w = order[0]
        gap = key[w] - key[order[1]] if kb > 1 and np.isfinite(key[order[1]]) else np.inf
        return int(d["cand"][w]), gap

    keep = d["keep"].copy()
    tok, gap = winner(keep)
    tp_margin = np.inf
    if d["topp"] > 0:
        for r in range(1, kb):
            m = abs(excl[r] - d["topp"])
            if m < 1e-4:
                flipped = keep.copy()
                flipped[r] = not flipped[r]
                if winner(flipped)[0] != tok:
                    tp_margin = min(tp_margin, m)
    return tp_margin, gap


def fast_row_gap(x_row, t, noise_row, draft=-1):
    """fp64 gap between the best and second-best fast-path scores of one row (inf when t <= 0:
    the plain argmax is exact)."""
    if not t > 0:
        return np.inf
    s = x_row.astype(np.float64) / float(t) + noise_row.astype(np.float64)
    if 0 <= draft < s.size:
        s[draft] = -np.inf
    top2 = -np.partition(-s, 1)[:2]
    if not np.isfinite(top2[0]) or not np.isfinite(top2[1]):
        return np.inf  # at most one finite score, or all -inf: ties go by token id exactly
    return float(top2[0] - top2[1])
