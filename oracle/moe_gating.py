"""ORACLE — test infrastructure only (never imported by the product).

MoE top-k gating (hpc.moe_topk_gating) in fp64: the contract of the operator's docstring, plus a
per-element bound on the kernel's fp32 weights and on its fp32 keys.

Ids follow the total order (key desc, id asc) with NaN below -inf, over the experts of the
topk_group best groups (group score desc, group id asc), and are compared exactly. A decision is
well posed when every pair of neighbours in that order (the k chosen experts and the next one; the
topk_group chosen groups and the next one) is either an exact tie of identical inputs, which the
kernel resolves the same way, or further apart than twice the sum of their error bounds
(`boundary_ok`); synth/moe_gating.py redraws inputs until it is.

Bounds, from the kernel's arithmetic (csrc/moe_gating.cu); u = 2^-24, gamma_d = d u / (1 - d u),
expf within 2 ulp (a relative 2^-22), / and + correctly rounded:

  * softmax: d_e = fl(x_e - m) is within u |x_e - m| of x_e - m, so expf(d_e) is within
    r1_e = (1 + 2^-22) exp(u |x_e - m|) - 1 of exp(x_e - m) (plus 2^-126 where it underflows).
    The sum: each lane adds at most 16 terms in order and a 5-level butterfly joins the lanes, at
    most 21 roundings: sigma = (1 + gamma_21)(1 + max r1 + E 2^-126) - 1 relative (the sum is
    >= 1: the maximum's term is exactly 1). s_e = fl(e_e / S): relative
    (1 + r1_e)(1 + u) / (1 - sigma) - 1, absolute 2^-125.
  * sigmoid: t = expf(-x) within 2^-22, fl(1 + t) and the divide one rounding each: relative
    (1 + u) / (1 - ((1 + 2^-22)(1 + u) - 1)) - 1, absolute 2^-126 (expf overflow gives 0).
  * key with a bias: fl(s + b), |err| <= err_s (1 + u) + u |c|.
  * group score: the max key (its error), or fl(k1 + k2): |err| <= (err_1 + err_2)(1 + u) + u |g|.
  * weights by interval arithmetic: w = s_id, or s_id / W with W summed over k in rank order
    (gamma_{k-1}), one rounding for the divide, one for the product with the scaling factor.
"""
import numpy as np

U = 2.0 ** -24
EXP_REL = 2.0 ** -22
TINY = 2.0 ** -149
FLOOR = 2.0 ** -126
SUM_DEPTH = 21  # 16 slots per lane + 5 butterfly levels


def _gamma(d):
    return d * U / (1 - d * U)


def _f64(a):
    import torch

    if isinstance(a, torch.Tensor):
        return a.detach().cpu().to(torch.float64).numpy()
    return np.asarray(a, np.float64)


def _order(keys, eligible=None):
    """Argsort of each row by (eligible first, NaN last among them, key desc, id asc)."""
    nan = np.isnan(keys)
    cls = nan.astype(np.int8)
    if eligible is not None:
        cls = np.where(eligible, cls, 2)
    neg = np.where(nan, 0.0, -keys)
    ids = np.broadcast_to(np.arange(keys.shape[-1]), keys.shape)
    return np.lexsort((ids, neg, cls), axis=-1)


def gating(logits, topk, scoring=0, renormalize=True, bias=None, num_expert_group=1,
           topk_group=1, routed_scaling_factor=1.0):
    """fp64 contract of hpc.moe_topk_gating on logits [T, E] (the values the kernel reads, i.e.
    fp32 or bf16 widened). Returns a dict: ids [T, k], weights [T, k], and the intermediate
    scores, keys, group scores, eligibility, orders and error bounds used by the checks."""
    x = _f64(logits)
    T, E = x.shape
    b = None if bias is None else _f64(bias).reshape(-1)
    f = float(np.float32(routed_scaling_factor))
    with np.errstate(all="ignore"):
        if scoring == 0:
            finite = np.where(np.isnan(x), -np.inf, x)
            m = finite.max(-1, keepdims=True) if E else np.zeros((T, 1))
            d = x - m
            e = np.exp(d)
            S = e.sum(-1, keepdims=True)
            s = e / S
            r1 = (1 + EXP_REL) * np.exp(U * np.abs(np.where(np.isfinite(d), d, 0.0))) - 1
            sigma = (1 + _gamma(SUM_DEPTH)) * (1 + r1.max(-1, keepdims=True) + E * FLOOR) - 1
            s_err = s * ((1 + r1) * (1 + U) / (1 - sigma) - 1) + 2 * FLOOR
        else:
            s = 1 / (1 + np.exp(-x))
            rho = (1 + EXP_REL) * (1 + U) - 1
            s_err = s * ((1 + U) / (1 - rho) - 1) + FLOOR
        if scoring == 0 and b is None:
            keys, k_err = x.copy(), np.zeros_like(x)
        else:
            keys = s + (0.0 if b is None else b)
            k_err = s_err * (1 + U) + (U * np.abs(keys) if b is not None else 0.0)
        eligible = np.ones((T, E), bool)
        G = num_expert_group
        g_scores = g_err = g_order = None
        if G > 1:
            gs = E // G
            kg = keys.reshape(T, G, gs)
            og = _order(kg)
            top = np.take_along_axis(kg, og[..., :2], -1)
            terr = np.take_along_axis(k_err.reshape(T, G, gs), og[..., :2], -1)
            if b is not None:
                g_scores = top[..., 0] + top[..., 1]
                g_err = (terr[..., 0] + terr[..., 1]) * (1 + U) + U * np.abs(g_scores)
            else:
                g_scores, g_err = top[..., 0], terr[..., 0]
            g_order = _order(g_scores)
            chosen_g = np.zeros((T, G), bool)
            np.put_along_axis(chosen_g, g_order[:, :topk_group], True, -1)
            eligible = np.repeat(chosen_g, gs, axis=-1)
        order = _order(keys, eligible)
        ids = order[:, :topk]
        w = np.take_along_axis(s, ids, -1)
        we = np.take_along_axis(s_err, ids, -1)
        lo, hi = np.maximum(w - we, 0.0), w + we
        if renormalize:
            W = w.sum(-1, keepdims=True)
            g = _gamma(max(topk - 1, 0))
            Wlo = (lo.sum(-1, keepdims=True)) * (1 - g)
            Whi = (hi.sum(-1, keepdims=True)) * (1 + g)
            w = w / W
            lo, hi = lo / Whi, hi / np.where(Wlo > 0, Wlo, np.nan)
        lo, hi = lo * (1 - U), hi * (1 + U)
        w = w * f
        lo, hi = np.sort(np.stack([lo * f * (1 - U), hi * f * (1 + U)]), axis=0)
        w_bound = np.maximum(hi - w, w - lo) + TINY * (1 + abs(f))
    return dict(ids=ids.astype(np.int32), weights=w, w_bound=w_bound, scores=s, keys=keys,
                key_err=k_err, eligible=eligible, order=order, group_scores=g_scores,
                group_err=g_err, group_order=g_order, x=x, bias=b)


def boundary_ok(ref, topk, topk_group=1, factor=2.0):
    """Per row: every neighbouring pair of the order, up to the first unchosen expert (and the
    first unchosen group), is an exact tie of identical inputs or more than `factor` times the sum
    of the two error bounds apart. Pairs with a NaN or an infinite key are exact ties or exact
    orders, so they pass."""
    x, b, keys, err = ref["x"], ref["bias"], ref["keys"], ref["key_err"]
    T, E = x.shape
    bb = np.zeros((T, E)) if b is None else np.broadcast_to(b, (T, E))
    n = min(topk + 1, E)
    o = ref["order"][:, :n]

    def pairs_ok(k, e, same):
        fin = np.isfinite(k[:, 1:]) & np.isfinite(k[:, :-1])
        far = np.abs(k[:, 1:] - k[:, :-1]) > factor * (e[:, 1:] + e[:, :-1])
        return (same | ~fin | far).all(-1)

    g = lambda a: np.take_along_axis(a, o, -1)  # noqa: E731
    xs, bs = g(x), g(bb)
    same = (xs[:, 1:] == xs[:, :-1]) & (bs[:, 1:] == bs[:, :-1])
    elig = g(ref["eligible"])
    same |= ~(elig[:, 1:] & elig[:, :-1])
    ok = pairs_ok(g(keys), g(err), same)
    if ref["group_scores"] is not None:
        gsc, gerr = ref["group_scores"], ref["group_err"]
        G = gsc.shape[1]
        gs = E // G
        go = ref["group_order"][:, :min(topk_group + 1, G)]
        gx = np.sort(x.reshape(T, G, gs), -1)
        gb = np.sort(bb.reshape(T, G, gs), -1)
        sel_x = np.take_along_axis(gx, go[..., None], 1)
        sel_b = np.take_along_axis(gb, go[..., None], 1)
        gsame = ((sel_x[:, 1:] == sel_x[:, :-1]).all(-1) & (sel_b[:, 1:] == sel_b[:, :-1]).all(-1))
        ok &= pairs_ok(np.take_along_axis(gsc, go, -1), np.take_along_axis(gerr, go, -1), gsame)
    return ok


def check(ids, weights, ref, rows=None):
    """The GPU test's check of one call against ref = gating(...) on the same rows: ids exactly,
    weights within the bound where the reference weight is finite, and every row's ids distinct
    and in [0, E). Returns a dict of failure counts (all must be 0)."""
    ids = np.asarray(ids.cpu() if hasattr(ids, "cpu") else ids).astype(np.int64)
    w = _f64(weights)
    if rows is not None:
        ids, w = ids[rows], w[rows]
    E = ref["x"].shape[1]
    rid, rw, rb = ref["ids"], ref["weights"], ref["w_bound"]
    fin = np.isfinite(rw)
    srt = np.sort(ids, -1)
    distinct = (srt[:, 1:] != srt[:, :-1]).all(-1) if ids.shape[1] > 1 else np.ones(len(ids), bool)
    return dict(ids=int((ids != rid).any(-1).sum()),
                range=int(((ids < 0) | (ids >= E)).any(-1).sum()),
                distinct=int((~distinct).sum()),
                weights=int((fin & ~(np.abs(w - rw) <= rb)).sum()))


def failed(res):
    return any(res.values())
