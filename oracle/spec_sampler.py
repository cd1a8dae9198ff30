"""numpy restatement of the fused speculative sampler (hpc.fused_speculative_sampler).

fp32 where the kernels round exactly (x / t, x / t + g, u * q), fp64 where they carry ulp-level
error (the softmax p, the residual log(p - q) + g). `mutations` names deliberate faults (see
MUTATIONS); tests use them to show that their inputs tell a correct sampler from a wrong one.
The Philox noise is oracle/sampler.py's; `philox_uniforms` adds the acceptance uniforms.
"""
import numpy as np

from oracle import sampler as osm

F32 = np.float32
NEG_INF = F32(-np.inf)

MUTATIONS = (
    "inverted_ratio",        # accept iff u * p(d) < q(d)
    "residual_unclamped",    # recovered token over every v of log|p - q| + g
    "bonus_from_prev_row",   # the bonus token drawn from row K - 1
    "q_next_position",       # q_i read from draft position i + 1
    "tie_larger_id",         # ties go to the larger token id
    "temperature_after_softmax",  # p = softmax(x) / t instead of softmax(x / t)
    "no_padding",            # out[b, n:] left 0 instead of -1
    "count_includes_bonus",  # num_accepted = accepted drafts + 1
    "draft_not_excluded",    # the rejected one-hot draft may be recovered
    "noise_of_request_row",  # noise row b instead of b * (K + 1) + j
)


def philox_uniforms(seed: int, offset: int, batch: int, k: int):
    """The kernel's acceptance uniforms [batch, k]: counter (0xFFFFFFFF, b * (k + 1) + i, offset lo,
    offset hi), key = seed, output word 0."""
    rows = (np.arange(batch)[:, None] * (k + 1) + np.arange(k)[None, :]).astype(np.uint32)
    ctr = np.zeros((batch, k, 4), np.uint32)
    ctr[..., 0] = np.uint32(0xFFFFFFFF)
    ctr[..., 1] = rows
    ctr[..., 2] = np.uint32(offset & 0xFFFFFFFF)
    ctr[..., 3] = np.uint32(offset >> 32)
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], np.uint32)
    return osm.uniform_from_bits(osm.philox4x32_10(ctr, key)[..., 0])


def argmax_id(key, larger=False):
    """(value desc, id asc) winner of a 1-D key; NaN never wins; 0 when no key is not NaN."""
    ok = ~np.isnan(key)
    if not ok.any():
        return 0
    best = key[ok].max()
    ties = np.nonzero(ok & (key == best))[0]
    return int(ties.max() if larger else ties.min())


def _gap(key):
    """fp64 distance from the best to the second-best finite key (inf if fewer than two)."""
    k = key[np.isfinite(key)]
    if k.size < 2:
        return np.inf
    top2 = -np.partition(-k, 1)[:2]
    return float(top2[0] - top2[1])


def _softmax64(xt):
    """p of fp32 rows xt [R, V] in fp64: exp(xt - max) / sum."""
    x = xt.astype(np.float64)
    m = x.max(axis=-1, keepdims=True)
    with np.errstate(invalid="ignore"):
        e = np.where(np.isneginf(x), 0.0, np.exp(x - m))
    return e / e.sum(axis=-1, keepdims=True)


def spec_sample(storage, vocab, draft_token_ids, *, draft_probs=None, temperature=0.0, uniform,
                noise, mutations=(), detail=False, eps=1e-4):
    """Returns (output_token_ids int32 [B, K + 1], num_accepted int32 [B][, details]).

    `storage` [B (K + 1), >= V] holds the logits as fp32 values; `uniform` [B, K] and `noise`
    [B (K + 1), V] fp32. With `detail`, per request: the acceptance margin (smallest
    |u q(d) - p(d)| / p(d) over the decided positions) and the key gap of the emitting row, made
    robust to a relative error `eps` of the kernel's p where the residual decides."""
    x_all = osm._rows(storage, vocab, mutations)
    d_all = np.asarray(draft_token_ids, np.int64)
    B, K = d_all.shape
    V = vocab
    temp = osm._per_row(temperature, B, np.float32)
    big = "tie_larger_id" in mutations
    out = np.full((B, K + 1), 0 if "no_padding" in mutations else -1, np.int32)
    nacc = np.zeros(B, np.int32)
    details = []
    for b in range(B):
        rows = x_all[b * (K + 1):(b + 1) * (K + 1)]
        d = d_all[b]
        t = temp[b]
        acc_margin, gap = np.inf, np.inf
        if not t > 0:
            a = [argmax_id(rows[i], big) for i in range(K + 1)]
            n = next((i for i in range(K) if d[i] != a[i]), K)
            tok = a[n]
        else:
            xt = (rows / F32(t)).astype(F32)
            p = _softmax64(rows.astype(np.float64)) / float(t) if "temperature_after_softmax" in mutations \
                else _softmax64(xt)
            n = K
            for i in range(K):
                if not 0 <= d[i] < V:
                    n = i
                    break
                qi = min(i + 1, K - 1) if "q_next_position" in mutations else i
                q = F32(1) if draft_probs is None else F32(draft_probs[b, qi, d[i]])
                u, pd = F32(uniform[b, i]), p[i, d[i]]
                uq = float(F32(u * q))
                acc_margin = min(acc_margin, abs(uq - pd) / pd if pd > 0 else np.inf)
                ok = float(F32(u * F32(pd))) < float(q) if "inverted_ratio" in mutations else uq < pd
                if not ok:
                    n = i
                    break
            j = K - 1 if (n == K and "bonus_from_prev_row" in mutations) else n
            r = b if "noise_of_request_row" in mutations else b * (K + 1) + j
            g = noise[r]
            plain = (xt[j] + g).astype(F32)
            if n < K and draft_probs is not None:
                qi = min(n + 1, K - 1) if "q_next_position" in mutations else n
                q = draft_probs[b, qi].astype(np.float64)
                pj = p[j]
                with np.errstate(divide="ignore", invalid="ignore"):
                    if "residual_unclamped" in mutations:
                        key = np.log(np.abs(pj - q)) + g
                    else:
                        key = np.where(pj > q, np.log(pj - q), -np.inf) + g
                    lo = np.where(pj * (1 - eps) > q, np.log(pj * (1 - eps) - q), -np.inf) + g
                    hi = np.where(pj * (1 + eps) > q, np.log(pj * (1 + eps) - q), -np.inf) + g
                if np.isfinite(key).any():
                    tok = argmax_id(key, big)
                    others = np.delete(hi, tok)
                    with np.errstate(invalid="ignore"):
                        gap = lo[tok] - (others.max() if others.size else -np.inf)
                else:  # empty residual: sample from p; robust only if no token can enter
                    tok = argmax_id(plain, big)
                    gap = _gap(plain.astype(np.float64)) if not np.isfinite(hi).any() else -np.inf
            else:
                key = plain.copy()
                if n < K and 0 <= d[n] < V and "draft_not_excluded" not in mutations:
                    key[d[n]] = NEG_INF
                tok = argmax_id(key, big)
                gap = _gap(key.astype(np.float64))
        out[b, :n] = d[:n]
        out[b, n] = tok
        nacc[b] = n + 1 if "count_includes_bonus" in mutations else n
        if detail:
            details.append(dict(n=n, acc_margin=acc_margin, gap=gap, sample=bool(t > 0)))
    return (out, nacc, details) if detail else (out, nacc)
