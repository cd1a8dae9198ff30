"""Seeded router logits for MoE top-k gating (hpc.moe_topk_gating), one builder per routing family,
and the same computation written as an fp32 torch chain (softmax / sigmoid -> topk -> gather ->
renormalize, vLLM's grouped_topk for groups), which tools/moe_gating_bench.py times.

Two kinds of input:
  * "random": rows redrawn until every decision clears the margins of oracle/moe_gating.py
    (`boundary_ok`): so a kernel whose expf differs from numpy's by an ulp cannot swap two ids;
  * "ties": a bias with repeated values, the same for every group, and in each row an exact tie
    planted across the k boundary (even rows) or two identical groups across the topk_group
    boundary (odd rows, grouped families): both must resolve to the lower id.
Special rows (`special_rows`): all NaN, all -inf, and a quarter of the columns at -inf.

The oracle is imported inside the builders that clear margins, so that the torch chain and the
plain builders stay importable without it.
"""
import zlib

import numpy as np
import torch

# family -> configuration of the routers the library is meant to serve
CONFIGS = {
    "mixtral": dict(E=8, topk=2, scoring=0, renormalize=True, bias=False, G=1, topk_group=1,
                    factor=1.0),
    "qwen3": dict(E=128, topk=8, scoring=0, renormalize=True, bias=False, G=1, topk_group=1,
                  factor=1.0),
    "deepseek_v2": dict(E=160, topk=6, scoring=0, renormalize=False, bias=False, G=8, topk_group=3,
                        factor=16.0),
    "deepseek_v3": dict(E=256, topk=8, scoring=1, renormalize=True, bias=True, G=8, topk_group=4,
                        factor=2.5),
    "kimi_k2": dict(E=384, topk=8, scoring=1, renormalize=True, bias=True, G=1, topk_group=1,
                    factor=2.827),
    "qwen3_next": dict(E=512, topk=10, scoring=0, renormalize=True, bias=False, G=1, topk_group=1,
                       factor=1.0),
}
# E not a multiple of the 16-byte vector: the last vector of a row is partly padding
ODD = dict(E=13, topk=3, scoring=1, renormalize=False, bias=True, G=1, topk_group=1, factor=1.0)
TRIES = 50


def seed_of(*key):
    return zlib.crc32(repr(key).encode()) % 100003


def hpc_kwargs(cfg, bias):
    """Keyword arguments of hpc.moe_topk_gating for a configuration."""
    return dict(topk=cfg["topk"], scoring=cfg["scoring"], renormalize=cfg["renormalize"],
                correction_bias=bias, num_expert_group=cfg["G"], topk_group=cfg["topk_group"],
                routed_scaling_factor=cfg["factor"])


def oracle(x, cfg, bias):
    from oracle import moe_gating as og

    return og.gating(x, cfg["topk"], cfg["scoring"], cfg["renormalize"], bias, cfg["G"],
                     cfg["topk_group"], cfg["factor"])


def _round(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dtype).float().numpy().astype(np.float64)


def make_bias(rng, cfg, kind):
    if not cfg["bias"]:
        return None
    E, G = cfg["E"], cfg["G"]
    if kind == "ties":  # coarse levels, the same pattern in every group
        pat = np.round(rng.normal(0.0, 0.1, E // G) * 8) / 8
        return np.tile(pat, G).astype(np.float32)
    return rng.normal(0.0, 0.1, E).astype(np.float32)


def _draw_row(rng, E, dtype):
    return _round(rng.standard_normal(E) * 2.0, dtype)


def _plant(x, ref, cfg, bias, t, group):
    """Plant a tie in row t of x (in place) from the row's oracle `ref` (one row). Returns
    (lower id, higher id, what) or None when the row has no candidate."""
    k, E = cfg["topk"], cfg["E"]
    bb = np.zeros(E) if bias is None else bias.astype(np.float64)
    if group:
        gs, tg = E // cfg["G"], cfg["topk_group"]
        A, B = ref["group_order"][0, tg - 1], ref["group_order"][0, tg]
        x[t, B * gs:(B + 1) * gs] = x[t, A * gs:(A + 1) * gs]
        return min(A, B), max(A, B), "group"
    o = ref["order"][0]
    a = o[k - 1]
    cand = [j for j in o[k:] if ref["eligible"][0, j] and bb[j] == bb[a]]
    if not cand:
        return None
    j = cand[0]
    x[t, j] = x[t, a]
    return min(a, j), max(a, j), "expert"


def _planted_ok(ref, cfg, p):
    lo, hi, what = p
    if what == "group":
        chosen = set(ref["group_order"][0, :cfg["topk_group"]].tolist())
    else:
        chosen = set(ref["ids"][0].tolist())
    return lo in chosen and hi not in chosen


def make_case(cfg, T, dtype=torch.float32, seed=0, kind="random", pad=0, rows=None):
    """One call's inputs. Returns dict(store: CPU tensor [T, E + pad] of `dtype` whose padding is
    +inf, logits: the view store[:, :E], x: its values in float64, bias: float32 tensor or None,
    cfg, planted: [(row, lower id, higher id, "expert" | "group")]). Only `rows` (default all) are
    cleared and planted: the others are plain draws that the test does not check."""
    from oracle import moe_gating as og

    rng = np.random.default_rng(seed)
    E = cfg["E"]
    bias = make_bias(rng, cfg, kind)
    x = np.stack([_draw_row(rng, E, dtype) for _ in range(T)]) if T else np.zeros((0, E))
    rows = np.arange(T) if rows is None else np.asarray(rows)
    planted = {}
    todo = rows
    for _ in range(TRIES):
        if kind == "ties":
            for t in todo:
                grp = cfg["G"] > 1 and t % 2 == 1
                p = _plant(x, oracle(x[t:t + 1], cfg, bias), cfg, bias, t, grp)
                if p is not None:
                    planted[int(t)] = p
        ref = oracle(x[todo], cfg, bias)
        ok = og.boundary_ok(ref, cfg["topk"], cfg["topk_group"])
        for i, t in enumerate(todo):
            if int(t) in planted:
                one = {k: (v[i:i + 1] if isinstance(v, np.ndarray) and v.ndim == 2 else v)
                       for k, v in ref.items()}
                ok[i] &= _planted_ok(one, cfg, planted[int(t)])
        todo = todo[~ok]
        if not len(todo):
            break
        for t in todo:
            x[t] = _draw_row(rng, E, dtype)
            planted.pop(int(t), None)
    else:
        raise ValueError(f"synth.moe_gating: {len(todo)} rows stay within the oracle's margin of a "
                         f"decision after {TRIES} draws")
    return _pack(x, cfg, dtype, bias, pad, [(t, *p) for t, p in sorted(planted.items())])


def _pack(x, cfg, dtype, bias, pad, planted):
    T, E = x.shape
    store = np.full((T, E + pad), np.inf, np.float32)
    store[:, :E] = x
    st = torch.from_numpy(store).to(dtype)
    return dict(store=st, logits=st[:, :E], x=st[:, :E].double().numpy(),
                bias=None if bias is None else torch.from_numpy(bias), cfg=cfg, planted=planted)


def special_rows(cfg, dtype=torch.float32, seed=0, pad=0):
    """Eight rows: all NaN, all -inf, a NaN among finite values, then rows with a quarter of the
    columns at -inf (never chosen while a finite key is available)."""
    rng = np.random.default_rng(seed)
    E = cfg["E"]
    bias = make_bias(rng, cfg, "random")
    x = np.stack([_draw_row(rng, E, dtype) for _ in range(8)])
    x[0] = np.nan
    x[1] = -np.inf
    x[2, rng.integers(E)] = np.nan
    from oracle import moe_gating as og

    for t in range(3, 8):  # the finite keys of these rows clear the margins
        for _ in range(TRIES):
            x[t, rng.choice(E, max(1, E // 4), replace=False)] = -np.inf
            ref = oracle(x[t:t + 1], cfg, None if bias is None else bias)
            if og.boundary_ok(ref, cfg["topk"], cfg["topk_group"])[0]:
                break
            x[t] = _draw_row(rng, E, dtype)
        else:
            raise ValueError(f"synth.moe_gating: special row {t} stays within the margin")
    return _pack(x, cfg, dtype, bias, pad, [])


def random_logits(T, E, dtype=torch.float32, seed=0, device="cpu", width=None):
    """Plain normal logits (x 2) for timing, optionally as the first E columns of [T, width]."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    full = (torch.randn((T, width or E), generator=g) * 2.0).to(dtype).to(device)
    return full[:, :E]


def torch_chain(logits, topk, scoring=0, renormalize=True, correction_bias=None,
                num_expert_group=1, topk_group=1, routed_scaling_factor=1.0):
    """The fp32 torch ops a caller writes without the fused kernel: softmax or sigmoid, the
    biased choice, vLLM's grouped_topk group mask, topk, gather, renormalize, scale."""
    x = logits.float()
    scores = torch.softmax(x, dim=-1) if scoring == 0 else torch.sigmoid(x)
    choice = scores if correction_bias is None else scores + correction_bias
    if num_expert_group > 1:
        T, E = x.shape
        grouped = choice.view(T, num_expert_group, E // num_expert_group)
        if correction_bias is None:
            gscore = grouped.max(dim=-1).values
        else:
            gscore = grouped.topk(2, dim=-1)[0].sum(dim=-1)
        gidx = torch.topk(gscore, k=topk_group, dim=-1, sorted=False)[1]
        gmask = torch.zeros_like(gscore).scatter_(1, gidx, 1)
        smask = gmask.unsqueeze(-1).expand(T, num_expert_group, E // num_expert_group).reshape(T, E)
        choice = choice.masked_fill(smask == 0, float("-inf"))
    ids = torch.topk(choice, k=topk, dim=-1)[1]
    w = scores.gather(1, ids)
    if renormalize:
        w = w / w.sum(dim=-1, keepdim=True)
    return ids.to(torch.int32), w * routed_scaling_factor
