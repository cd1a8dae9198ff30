"""fp64 oracle of the route GEMM (csrc/gemm_bf16xfp32.cu) and the stand-alone grouped FP8 GEMMs
(csrc/group_gemm_fp8.cu, csrc/activation.cu, csrc/fuse_moe.cu reformat_x_scale_kernel), with
per-element bounds derived from the kernels' arithmetic, in the manner of oracle/moe_exact.py.

Tensor-core accumulation (all three kernels). Products of bf16 x bf16 and of e4m3 x e4m3 (converted
to fp16, exactly) are exact in fp32. How Hopper's tensor cores add them inside a wgmma chain is not
documented, so the bound is a stated model, not a derivation: every fp32 add of a chain of length
K_chain may truncate, i.e. err by 2^-23 of a partial sum, and every partial sum is at most
S = sum |a w| over the chain. So a chain's value errs by at most K_chain 2^-23 S. `route_accumulation_ratio`
measures (actual error) / E directly on the route GEMM's fp32 output; the model requires <= 1.

Route GEMM, split s of `split` (gemm_bf16xfp32.cu:69-73 and 110-168). The K steps of 64 columns are
dealt out ceil(steps / split) per CTA of the cluster, so the last CTAs get fewer, or none. Per
split the kernel chains hi_s = X.W_high^T and lo_s = X.W_low^T over that split's K_s columns (a ragged
last step is TMA zero-fill: K_chain = 64 * steps), forms t_s = hi_s + scale lo_s (a product and an
add, or one fma: two fp32 roundings at most, each 2^-24 of at most S_s = S_high,s + |scale| S_low,s),
and the cluster sums t_0 + ... + t_{split-1} in split order in fp32 (split - 1 adds, each 2^-24 of at
most S = sum_s S_s). So
  E = sum_s (K_chain,s 2^-23 + 2 2^-24) S_s + (split - 1) 2^-24 S
and the fp32 output is within E of y = X.(W_high + scale W_low)^T. The bf16 output is one
round-to-nearest of that value: B = 2^-8 (|y| + E) + E. `|scale|` multiplies the low chain's S.

Per-tensor grouped GEMM (group_gemm_fp8_kernel<false, false>): one fp16 wgmma accumulator chained
over all ceil(K/128) K blocks of 128 (a ragged last block is TMA zero-fill), then acc *= y_scale[g]
(one fp32 rounding) and a bf16 round-to-nearest:
  E = |ys| Kpad 2^-23 S + 2^-24 (|y| + |ys| Kpad 2^-23 S),   B = 2^-8 (|y| + E) + E.

Blockwise grouped GEMM (group_gemm_fp8_kernel<true, false>): moe_exact._gemm_rows (a fresh 128-term
accumulator per K block, promoted by fmaf with fl32(xs ws)), B = 2^-8 (|y| + E) + E. The activation
scale of row i of group g is column pad_base[g] + i of the transposed layout, where pad_base is the
exclusive sum of each group's rows rounded up to the granule `scale_granule(avg)` (the bucket rule is
written out in moe_exact.scale_granule, not taken from the library). The weight scale of (g, n, kb)
is w_scale[g, n // 128, kb]; the kpad4 - K/128 padding entries are never read.

reformat_x_scale is a pure copy: `reformat_layout` is exact, and leaves every column it does not
write NaN so that a comparison sees a write in the wrong place.

The fp32 emulations `route_emulate` and `grouped_emulate` restate the kernels' arithmetic in torch
fp32 and take named bugs (ROUTE_BUGS, GROUPED_BUGS); tests/test_gemm_exact_cpu.py shows the checks
pass the emulation and catch every bug.
"""
import torch

from oracle import moe_exact as ox
from oracle.moe_exact import BF16_HALF_ULP_REL, check_down, round_sig  # noqa: F401  (re-exported)

ACC_ULP = 2.0 ** -23
U32 = 2.0 ** -24
ROUTE_BM, ROUTE_BK = 128, 64
GROUP_BM, GROUP_BK = 64, 128


# ------------------------------------------------------------------------------------------------
# route GEMM
# ------------------------------------------------------------------------------------------------
def route_splits(k, split):
    """[(k0, k1, steps)] per CTA of the cluster: the K columns [k0, k1) it reads (clipped to k) and
    its number of 64-column steps (0 for a CTA with nothing to do)."""
    total = (k + ROUTE_BK - 1) // ROUTE_BK
    per = (total + split - 1) // split
    out = []
    for s in range(split):
        n = max(0, min(per, total - s * per))
        k0 = min(k, s * per * ROUTE_BK)
        out.append((k0, min(k, k0 + n * ROUTE_BK), n))
    return out


def route_tile_n(n):
    return 128 if n % 128 == 0 else 64


def route_exact(x, w_high, w_low, scale, split, rows=None):
    """y = X.(W_high + scale W_low)^T in fp64 for `rows` of x (all if None), the bf16 bound B and the
    fp32 bound E of the module docstring (both [nr, n])."""
    X = (x if rows is None else x[rows]).double()
    Wh, Wl = w_high.double(), w_low.double()
    y = X @ Wh.t() + scale * (X @ Wl.t())
    E = torch.zeros_like(y)
    S_all = torch.zeros_like(y)
    for k0, k1, steps in route_splits(x.size(1), split):
        if steps == 0:
            continue
        Xa = X[:, k0:k1].abs()
        S = Xa @ Wh[:, k0:k1].abs().t() + abs(scale) * (Xa @ Wl[:, k0:k1].abs().t())
        E += (steps * ROUTE_BK * ACC_ULP + 2 * U32) * S
        S_all += S
    E += (split - 1) * U32 * S_all
    return y, BF16_HALF_ULP_REL * (y.abs() + E) + E, E


def route_accumulation_ratio(out_fp32, y, E):
    """Worst |out - y| / E of the route GEMM's fp32 output: the accumulation error measured against
    the model's E (<= 1 where the model holds). Raises if it exceeds 1."""
    err = (out_fp32.double() - y).abs()
    assert torch.isfinite(err).all(), "route: non-finite fp32 output"
    ratio = torch.where(err == 0, torch.zeros_like(err), err / E)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    assert worst <= 1.0, f"route fp32: |out - y| / E = {worst:.3g} at {int(ratio.argmax())}"
    return worst


def check_route(out, y, B, E, fp32_out, tag="route"):
    """Grade the route GEMM's rows `out` ([nr, n]); returns (worst err/B, accumulation ratio)."""
    if fp32_out:
        r = route_accumulation_ratio(out, y, E)
        return r, r
    return check_down(out, y, B, tag), ox.accumulation_probe(out, y, B, tag)


ROUTE_BUGS = ("no_low", "scale_ignored", "scale_twice", "drop_last_kstep", "k_tail_next_row",
              "split_missing", "split_doubled", "m_tail_last_row", "tile_n64_shift", "lanes_swapped",
              "bf16_truncate")


def _last_busy_split(k, split):
    return max(s for s, (_, _, steps) in enumerate(route_splits(k, split)) if steps)


def route_bug_expressible(bug, m, n, k, scale, split, fp32_out):
    """Whether a case can show `bug` at all (the bug changes nothing otherwise)."""
    return {"no_low": True,
            "scale_ignored": scale != 1.0,
            "scale_twice": abs(scale) != 1.0,
            "drop_last_kstep": True,
            "k_tail_next_row": k % ROUTE_BK != 0,
            "split_missing": _last_busy_split(k, split) > 0,
            "split_doubled": _last_busy_split(k, split) > 0,
            "m_tail_last_row": m % ROUTE_BM != 0,
            "tile_n64_shift": route_tile_n(n) == 64 and n > 64,
            "lanes_swapped": True,
            "bf16_truncate": not fp32_out}[bug]


def _bf16_truncate(v):
    return (v.float().contiguous().view(torch.int32) & -65536).view(torch.float32).to(torch.bfloat16)


def route_emulate(x, w_high, w_low, scale, split, fp32_out, rows=None, bug=None):
    """The route kernel's arithmetic in torch fp32 for `rows` (all if None), with an optional named
    bug from ROUTE_BUGS. Returns [nr, n] fp32 or bf16."""
    m, k = x.shape
    n = w_high.size(0)
    rows = torch.arange(m) if rows is None else rows
    steps = (k + ROUTE_BK - 1) // ROUTE_BK
    kpad = steps * ROUTE_BK

    def padded(t, idx):
        # the TMA box of the last step reads zeros past k; the bug reads on into the next rows
        if bug == "k_tail_next_row":
            flat = torch.cat([t.reshape(-1).float(), torch.zeros(kpad)])
            return flat[idx[:, None] * k + torch.arange(kpad)[None]]
        p = torch.zeros(idx.numel(), kpad)
        p[:, :k] = t[idx].float()
        return p

    X = padded(x, rows)
    cols = torch.arange(n)
    if bug == "tile_n64_shift" and route_tile_n(n) == 64:
        cols = (cols + 64) % n  # column tile nt reads the weights of tile nt + 1
    Wh, Wl = padded(w_high, cols), padded(w_low, cols)
    parts = []
    for s, (k0, _, st) in enumerate(route_splits(k, split)):
        a, b = k0, k0 + st * ROUTE_BK
        if bug == "drop_last_kstep" and b == kpad and st:
            b -= ROUTE_BK
        hi = X[:, a:b] @ Wh[:, a:b].t()
        lo = X[:, a:b] @ Wl[:, a:b].t()
        sc = {"no_low": 0.0, "scale_ignored": 1.0, "scale_twice": scale * scale}.get(bug, scale)
        parts.append(hi + torch.tensor(sc, dtype=torch.float32) * lo)
    last = _last_busy_split(k, split)
    acc = torch.zeros(rows.numel(), n)
    for s, t in enumerate(parts):
        if bug == "split_missing" and s == last and s > 0:
            continue
        acc = acc + t
        if bug == "split_doubled" and s == last and s > 0:
            acc = acc + t
    if bug == "lanes_swapped":
        acc = acc.view(-1, n // 4, 4)[..., [1, 0, 2, 3]].reshape(-1, n)
    out = acc if fp32_out else (_bf16_truncate(acc) if bug == "bf16_truncate" else acc.to(torch.bfloat16))
    if bug == "m_tail_last_row" and m % ROUTE_BM:
        out[rows == m - 1] = float("nan")
    return out


# ------------------------------------------------------------------------------------------------
# grouped FP8 GEMMs
# ------------------------------------------------------------------------------------------------
def pad_base(seqlens, granule):
    """First activation-scale column of every group: exclusive sum of rows rounded up to granule."""
    padded = (seqlens.long() + granule - 1) // granule * granule
    base = torch.zeros(seqlens.numel(), dtype=torch.long)
    base[1:] = torch.cumsum(padded, 0)[:-1]
    return base


def reformat_layout(x_scale, seqlens, cu_seqlens, tile):
    """Exact output of reformat_x_scale: row-major x_scale [m, KB] -> [KB, m] with group g's rows at
    columns pad_base[g] ..; every other column NaN. (Wider than m where the padded groups do not fit
    in m columns: the kernel's output is [KB, m], so callers keep every group within m / G rows.)"""
    m, kb = x_scale.shape
    base = pad_base(seqlens, tile)
    width = max(m, int(base[-1]) + int(seqlens[-1])) if seqlens.numel() else m
    out = torch.full((kb, width), float("nan"))
    for g in range(seqlens.numel()):
        n, r0 = int(seqlens[g]), int(cu_seqlens[g])
        out[:, int(base[g]):int(base[g]) + n] = x_scale[r0:r0 + n].t().float()
    return out


def group_rows(seqlens, cu_seqlens, row_start=None):
    """(group, index in group) of every row that belongs to a group, as two [M]-sized maps with -1
    elsewhere; `row_start` overrides cu_seqlens as the first row of each group."""
    starts = cu_seqlens[:-1] if row_start is None else row_start
    M = int(max([int(starts[g]) + int(seqlens[g]) for g in range(seqlens.numel())] + [0]))
    gi = torch.full((M,), -1, dtype=torch.long)
    ii = torch.full((M,), -1, dtype=torch.long)
    for g in range(seqlens.numel()):
        n, r0 = int(seqlens[g]), int(starts[g])
        gi[r0:r0 + n] = g
        ii[r0:r0 + n] = torch.arange(n)
    return gi, ii


def rows_to_check(seqlens, cu_seqlens, n, k, tile_m=GROUP_BM, granule=None, seed=0, n_random=4,
                  small=1 << 24):
    """Every row of every group when rows * n * k is small; otherwise moe_exact.rows_to_check's rows
    (first and last of each group, both sides of every tile and granule boundary, a seeded sample)."""
    rows_total = int(seqlens.sum())
    if rows_total * n * k <= small:
        gi, _ = group_rows(seqlens, cu_seqlens)
        return (gi >= 0).nonzero().flatten()
    r = dict(counts=seqlens.to(torch.int32), cu=cu_seqlens, granule=granule or tile_m)
    return ox.rows_to_check(r, seed=seed, n_random=n_random, tile_m=tile_m)


def route_rows(m, n, k, seed=0, n_random=8, small=1 << 24):
    """Rows of the route GEMM to grade: all when m * n * k is small, else every 128-row boundary."""
    if m * n * k <= small:
        return torch.arange(m)
    return rows_to_check(torch.tensor([m]), torch.tensor([0, m]), n, k, tile_m=ROUTE_BM, seed=seed,
                         n_random=n_random, small=0)


def _owners(seqlens, cu_seqlens, rows):
    gi, ii = group_rows(seqlens, cu_seqlens)
    g, i = gi[rows], ii[rows]
    assert (g >= 0).all(), "rows outside every group have no oracle value"
    return g, i


def grouped_pertensor_exact(x, w, seqlens, cu_seqlens, y_scale, rows=None):
    """fp64 y, bound B and pre-rounding bound E ([nr, N]) of the per-tensor grouped GEMM for `rows`
    (every row of every group if None)."""
    if rows is None:
        rows = rows_to_check(seqlens, cu_seqlens, 1, 1)
    g_of, _ = _owners(seqlens, cu_seqlens, rows)
    kpad = (x.size(1) + GROUP_BK - 1) // GROUP_BK * GROUP_BK
    y = torch.empty((rows.numel(), w.size(1)), dtype=torch.float64)
    E = torch.empty_like(y)
    for g in torch.unique(g_of).tolist():
        sel = (g_of == g).nonzero().flatten()
        A, W = x[rows[sel]].double(), w[g].double()
        ys = float(y_scale[g])
        v = ys * (A @ W.t())
        chain = abs(ys) * kpad * ACC_ULP * (A.abs() @ W.abs().t())
        y[sel] = v
        E[sel] = chain + U32 * (v.abs() + chain)
    return y, BF16_HALF_ULP_REL * (y.abs() + E) + E, E


def grouped_blockwise_exact(x, w, seqlens, cu_seqlens, xscale_t, w_scale, granule, rows=None):
    """fp64 y, bound B and E ([nr, N]) of the blockwise grouped GEMM, reading the activation scale of
    (g, i) from column pad_base[g] + i of xscale_t [KB, m_pad]."""
    if rows is None:
        rows = rows_to_check(seqlens, cu_seqlens, 1, 1)
    g_of, i_of = _owners(seqlens, cu_seqlens, rows)
    base = pad_base(seqlens, granule)
    y = torch.empty((rows.numel(), w.size(1)), dtype=torch.float64)
    E = torch.empty_like(y)
    for g in torch.unique(g_of).tolist():
        sel = (g_of == g).nonzero().flatten()
        v, e = ox._gemm_rows(x[rows[sel]], w[g], xscale_t[:, base[g] + i_of[sel]], w_scale[g])
        y[sel], E[sel] = v, e
    return y, BF16_HALF_ULP_REL * (y.abs() + E) + E, E


GROUPED_BUGS = ("yscale_neighbour", "rows_from_seqlens_prefix", "drop_last_kblock",
                "subnormal_as_normal", "reformat_granule", "wscale_stride_kb", "act_scale_next_row",
                "scatter_off_by_one")


def reformat_granule_old(avg):
    """The granule rule reformat_x_scale used before it shared the GEMM's: 64 for every avg > 48."""
    for top in (8, 16, 32, 48):
        if avg <= top:
            return top
    return 64


def _decode_e4m3(t, bug):
    v = t.float()
    if bug == "subnormal_as_normal":
        b = t.view(torch.uint8).to(torch.int32)
        sub = ((b & 0x78) == 0) & ((b & 7) != 0)
        as_normal = (1 + (b & 7).float() / 8) * 2.0 ** -6 * torch.where(b >= 0x80, -1.0, 1.0)
        v = torch.where(sub, as_normal, v)
    return v


def grouped_emulate(x, w, seqlens, cu_seqlens, rows, y_scale=None, xscale_t=None, w_scale=None,
                    avg=None, bug=None):
    """The grouped kernel's arithmetic in torch fp32 for output `rows`: per-tensor when y_scale is
    given, blockwise otherwise. Rows the (possibly buggy) kernel would not write come back NaN.
    Returns [nr, N] bf16."""
    G, N, K = w.shape
    starts = cu_seqlens[:-1]
    if bug == "rows_from_seqlens_prefix":
        starts = torch.zeros(G, dtype=torch.long)
        starts[1:] = torch.cumsum(seqlens.long(), 0)[:-1]
    gi, ii = group_rows(seqlens, cu_seqlens, starts)
    inside = rows < gi.numel()
    g_of = torch.full_like(rows, -1)
    i_of = torch.full_like(rows, -1)
    g_of[inside], i_of[inside] = gi[rows[inside]], ii[rows[inside]]
    KB = (K + GROUP_BK - 1) // GROUP_BK
    kpad = KB * GROUP_BK
    used = (KB - 1) * GROUP_BK if bug == "drop_last_kblock" else kpad
    out = torch.full((rows.numel(), N), float("nan"))
    for g in torch.unique(g_of).tolist():
        if g < 0:
            continue
        sel = (g_of == g).nonzero().flatten()
        A = torch.zeros(sel.numel(), kpad)
        A[:, :K] = _decode_e4m3(x[rows[sel]], bug)
        W = torch.zeros(N, kpad)
        W[:, :K] = _decode_e4m3(w[g], bug)
        if y_scale is not None:
            gs = g
            if bug == "yscale_neighbour":
                gs = g + 1 if g + 1 < G else g - 1
            out[sel] = (A[:, :used] @ W[:, :used].t()) * y_scale[gs].float()
            continue
        gran = (reformat_granule_old if bug == "reformat_granule" else ox.scale_granule)(avg)
        cols = pad_base(seqlens, gran)[g] + i_of[sel] + (1 if bug == "act_scale_next_row" else 0)
        # a column past the layout reads NaN
        xs_ext = torch.cat([xscale_t.float(), torch.full((xscale_t.size(0), 1), float("nan"))], 1)
        xs = xs_ext[:, cols.clamp(max=xscale_t.size(1))]  # [KB, nr]
        stride = KB if bug == "wscale_stride_kb" else w_scale.size(2)
        flat = w_scale.reshape(-1).float()
        acc = torch.zeros(sel.numel(), N)
        for kb in range(used // GROUP_BK):
            P = A[:, kb * 128:(kb + 1) * 128] @ W[:, kb * 128:(kb + 1) * 128].t()
            ws = flat[(g * (N // 128) + torch.arange(N) // 128) * stride + kb]
            acc = acc + P * (xs[kb][:, None] * ws[None])
        out[sel] = acc
    return out.to(torch.bfloat16)


def scatter_rows(row_indices, pool_rows, bug=None):
    """The pool row gather_rows_kernel copies for each problem row: indices are clamped into
    [0, pool_rows) (activation.cu gather_rows_kernel)."""
    idx = row_indices.long() + (1 if bug == "scatter_off_by_one" else 0)
    return idx.clamp(0, pool_rows - 1)
