"""Seeded inputs for the fused sampler: logits families, penalty masks, per-row parameters, and Gumbel
noise redrawn row by row until every row clears the margins of oracle/sampler.py (fp64): so a
sampler whose exp/log differ from numpy's by an ulp cannot flip a token.
"""
import zlib

import numpy as np
import torch

from oracle import sampler as osm

FAMILIES = ("normal", "peaked", "ties", "ascending", "descending", "constant", "sparse", "all_neg_inf")
MARGIN = 1e-4


def _family_row(rng, fam, V, max_topk):
    if fam == "normal":
        return rng.standard_normal(V) * 2.0
    if fam == "peaked":  # a few dominant tokens: top-p cuts at rank 2-5
        r = rng.standard_normal(V)
        top = rng.choice(V, 5, replace=False)
        r[top] = 14.0 - np.arange(5) * rng.uniform(0.3, 1.2)
        return r
    if fam == "ties":  # coarse levels: exact ties straddle the K boundary, also in bf16
        r = np.floor(rng.standard_normal(V) * 2.0) / 2.0
        r[rng.choice(V, 3 * max_topk, replace=False)] = 5.0
        return r
    if fam == "ascending":
        return np.linspace(-6.0, 6.0, V)
    if fam == "descending":
        return np.linspace(6.0, -6.0, V)
    if fam == "constant":
        return np.ones(V)
    if fam == "sparse":  # fewer finite values than K
        r = np.full(V, -np.inf)
        k = int(rng.integers(1, max_topk // 2))
        r[rng.choice(V, k, replace=False)] = rng.standard_normal(k) * 2.0
        return r
    return np.full(V, -np.inf)


def gumbel(rng, shape):
    u = rng.uniform(size=shape).astype(np.float32)
    u = np.clip(u, np.float32(2.0 ** -24), np.float32(1 - 2.0 ** -24))
    return osm.gumbel_from_uniform(u)


def make_logits(rng, B, V, dtype, pad, max_topk, families=FAMILIES):
    """Storage [B, V + pad] (padding +inf: never to be read) as float32 numpy and as a torch tensor
    of `dtype`, plus the family of every row."""
    fams = [families[b % len(families)] for b in range(B)]
    rows = np.stack([_family_row(rng, f, V, max_topk) for f in fams]) if B else np.zeros((0, V))
    store = np.full((B, V + pad), np.inf, np.float32)
    store[:, :V] = rows
    t = torch.from_numpy(store).to(dtype)
    return t.float().numpy(), t, fams


def _draw(rng, kind, B, choices, dtype):
    vals = rng.choice(np.asarray(choices), B)
    return vals.astype(dtype) if kind == "tensor" else vals[0].item() if B else choices[0]


def make_full_case(seed, B, V, dtype=torch.bfloat16, max_topk=32, policy=2, pad=0,
                   forms="tensor", topk_dtype=np.int64, penalty=True, families=FAMILIES):
    """One full-path call: the numpy inputs (`np`), the logits storage as a CPU tensor of `dtype`
    (`store_t`) and each row's family (`fams`), noise already redrawn for the margins. `forms` is
    "tensor" or "scalar" for every per-row parameter."""
    rng = np.random.default_rng(seed)
    store, store_t, fams = make_logits(rng, B, V, dtype, pad, max_topk, families)
    max_bs = B + 3
    mask = slot = None
    rp = 0.0
    if penalty:
        mask = (rng.uniform(size=(max_bs, V // 8, 8)) < 0.05)
        mask = np.packbits(mask, axis=-1, bitorder="little")[..., 0].astype(np.uint8)
        slot = rng.permutation(max_bs)[:B].astype(np.int32)
        rp = _draw(rng, forms, B, [0.0, 1.3, 1.05, 2.0], np.float32)
    temp = _draw(rng, forms, B, [0.0, 0.7, 1.0, 1.5], np.float32)
    topk = _draw(rng, forms, B, [0, 1, 20, max_topk, max_topk + 5], topk_dtype)
    if policy:
        topp = _draw(rng, forms, B, [0.0, 0.3, 0.8, 0.9, 1.0], np.float32)
        if forms == "scalar" and topp == 0.0:
            topp = 0.9
        if forms == "scalar" and topk == 0:
            topk = 20
    else:
        topp = 0.0
    noise = gumbel(rng, (B, V))
    kw = dict(penalty_mask=mask, slot_id=slot, repetition_penalty=rp, temperature=temp,
              softmax_policy=policy, topk=topk, topp=topp, max_topk=max_topk)
    for b in range(B):
        _redraw_until(lambda: full_row_ok(store, V, kw, noise, b), noise, b, rng, f"full-path row {b} ({fams[b]})")
    return dict(np=dict(store=store, V=V, noise=noise, **kw), store_t=store_t, fams=fams)


def _redraw_until(ok, noise, b, rng, what, tries=50):
    """Redraw row b of `noise` until ok() holds; a row that never clears the margins is an error, not
    a row to compare anyway."""
    for _ in range(tries):
        if ok():
            return
        noise[b] = gumbel(rng, noise.shape[1])
    raise ValueError(f"synth.sampler: {what} stays within {MARGIN} of a rounding decision after "
                     f"{tries} noise draws")


def _row_kw(kw, b):
    out = dict(kw)
    for k in ("repetition_penalty", "temperature", "topk", "topp"):
        if isinstance(kw[k], np.ndarray):
            out[k] = kw[k][b:b + 1]
    if kw["slot_id"] is not None:
        out["slot_id"] = kw["slot_id"][b:b + 1]
    return out


def full_row_margins(store, V, kw, noise, b):
    _, _, det = osm.fused_sampler(store[b:b + 1], V, noise=noise[b:b + 1], detail=True, **_row_kw(kw, b))
    return osm.row_margins(det[0])


def full_row_ok(store, V, kw, noise, b):
    tp, gap = full_row_margins(store, V, kw, noise, b)
    return tp >= MARGIN and gap >= MARGIN


def make_fast_case(seed, B, V, dtype=torch.bfloat16, pad=0, forms="tensor", draft=True,
                   families=FAMILIES):
    """One temperature-only call, as make_full_case; with `forms` "tensor" some rows have t = 0, -1 or
    NaN (greedy rows)."""
    rng = np.random.default_rng(seed)
    store, store_t, fams = make_logits(rng, B, V, dtype, pad, 32, families)
    temp = _draw(rng, forms, B, [0.0, -1.0, np.nan, 0.7, 1.0, 1.5] if forms == "tensor" else [0.7], np.float32)
    d = None
    if draft:
        d = rng.choice(np.array([-1, 0, 5, V - 1, V, V + 100, -7]), B).astype(np.int64)
        hit = rng.uniform(size=B) < 0.3  # some rows mask their current best token
        t = np.broadcast_to(np.asarray(temp, np.float32), (B,))
        for b in np.nonzero(hit)[0]:
            d[b] = int(np.argmax(store[b, :V] / (t[b] if t[b] > 0 else 1.0)))
    noise = gumbel(rng, (B, V))
    tt = np.broadcast_to(np.asarray(temp, np.float32), (B,))
    for b in range(B):
        _redraw_until(lambda: osm.fast_row_gap(store[b, :V], tt[b], noise[b],
                                               -1 if d is None else int(d[b])) >= MARGIN,
                      noise, b, rng, f"fast-path row {b} ({fams[b]})")
    return dict(np=dict(store=store, V=V, noise=noise, temperature=temp, draft_token_ids=d),
                store_t=store_t, fams=fams)


# The GPU test's grid: (dtype, B, V, max_topk, policy, forms) for the full path and
# (dtype, B, V, forms) for the temperature-only path, each case built by full_case / fast_case.
BIG_V = (120832, 151936)
FULL_GRID = (
    [(dt, 4, V, mk, pol, "tensor") for dt in ("fp32", "bf16") for V in (4096, 120832)
     for mk in (32, 64) for pol in (0, 1, 2)]
    + [(dt, B, V, 32, 2, forms) for dt in ("fp32", "bf16") for B in (1, 64, 512) for V in BIG_V
       for forms in ("tensor", "scalar")]
    + [("bf16", 64, 151936, 64, pol, "tensor") for pol in (0, 1)]
)
FAST_GRID = ([(dt, B, V, "tensor") for dt in ("fp32", "bf16") for B in (1, 4, 64, 512)
              for V in (4096,) + BIG_V] + [(dt, 64, 120832, "scalar") for dt in ("fp32", "bf16")])


def _seed(*key):
    return zlib.crc32(repr(key).encode()) % 100003


def _torch_dtype(dt):
    return torch.float32 if dt == "fp32" else torch.bfloat16


def full_case(dt, B, V, max_topk, policy, forms):
    """The FULL_GRID case: +inf row padding of 4 or 256 (fp32, odd / even B) or 128 (bf16), topk in
    int32 for odd B and int64 for even B."""
    pad = (4 if B % 2 else 256) if dt == "fp32" else 128
    return make_full_case(_seed(dt, B, V, max_topk, policy, forms), B, V, dtype=_torch_dtype(dt),
                          max_topk=max_topk, policy=policy, pad=pad, forms=forms,
                          topk_dtype=np.int32 if B % 2 else np.int64)


def fast_case(dt, B, V, forms):
    """The FAST_GRID case: +inf row padding of 256 (fp32) or 128 (bf16)."""
    return make_fast_case(_seed(dt, B, V, forms), B, V, dtype=_torch_dtype(dt),
                          pad=256 if dt == "fp32" else 128, forms=forms)
