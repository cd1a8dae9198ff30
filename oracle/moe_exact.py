"""Stage-by-stage fp64 oracle of the blockwise FusedMoE pipeline, with error bounds derived from the
kernels' own arithmetic (csrc/fuse_moe.cu, csrc/group_gemm_fp8.cu).

Each stage is computed from the kernel's own inputs to that stage (the gathered rows and scale
layout the route kernel wrote, the codes and scales the Gate-Up epilogue wrote, the bf16 rows the
Down GEMM wrote), so no stage inherits an earlier stage's rounding.

route (exact). counts / cu / topk_pos follow the deterministic order of moe_route_gather_kernel:
experts in order, and inside an expert the flattened (token, k) order. The activation-scale layout
[H/128, num_padded] puts row j of expert e at column pad_base[e] + j, where pad_base is the
exclusive sum of each expert's row count rounded up to the scale granule. The granule is picked
from avg = T*K // E_total by the bucket rule of `scale_granule` below (written out here, not taken
from the library).

GEMM arithmetic (both GEMMs). For a row r and an output column n, K block kb (128 products):
  P_kb  = sum_k a_k w_k: e4m3 x e4m3 products are exact in fp16/fp32; the fp16 wgmma adds them in
          an fp32 accumulator. How Hopper's tensor cores add inside a wgmma is not documented, so
          F16_ACC_EPS is a model, not a derivation: an fp32 adder that truncates, whose error over a
          128-term sum is at most 127 * 2^-23 * S_kb, S_kb = sum_k |a_k w_k|; F16_ACC_EPS = 2^-16
          (= 128 * 2^-23). `accumulation_probe` measures it (see below).
  f_kb  = fl32(xs * ws): one fp32 rounding, 2^-24 relative;
  acc  += fl32(P_kb * f_kb) by fmaf: one rounding per K block, <= 2^-24 * sum |f P|.
So the pre-rounding GEMM value v has |v - v_exact| <= E = sum_kb |f_kb| F16_ACC_EPS S_kb
+ (KB + 1) 2^-24 sum_kb |f_kb P_kb|.

Gate-Up epilogue (per row, per 128-column block of I): g, u = bf16_rn(v) for gate and up;
a = silu(g) * u in fp32 (silu = __fdividef(x, 1 + __expf(-x))); s = amax|a| / 448; codes =
e4m3_rn(a * (1 / (s + 1e-8))). The oracle follows the same chain from the exact v. A code may differ
from the oracle's by one step only where that is explained:
  (i)  g or u lies within E of a bf16 rounding boundary (bf16_rn(v - E) != bf16_rn(v + E)), or
  (ii) a * inv lies within ACT_REL of the boundary between the two codes. ACT_REL = 2^-18 covers
       __expf (2 + 1.16|x| ulp for the |x| < 16 that occur here), __fdividef (2 ulp), the product and
       a possibly approximate reciprocal (1 ulp): < 2^5 ulp of fp32.
The block scale times 448 must lie in the range the block's amax can take when every g and u takes
either of the bf16 roundings its bound E leaves open (widened by ACT_REL); outside rounding
ambiguities that range is the single oracle value (up to the fp32 division by 448). Oracle codes
are recomputed with the kernel's own scale, so a flipped amax does not cascade into the block.

Down (bf16 output): |out - y_exact| <= B = 2^-8 (|y_exact| + E) + E, the first term being bf16
round-to-nearest (half an ulp of 8 significant bits).

reduce: out[t] = bf16_rn(sum_k w_k x_k + shared) with fp32 products and sums in k order; bound
B = 2^-8 (|o| + E) + E with E = (K + 2) 2^-24 sum |terms| (one rounding per product and per add).

err/B of a bf16 output is dominated by the half-ulp term, so it cannot tell whether E is adequate.
`accumulation_probe` isolates E: wherever the kernel's bf16 value is not bf16_rn(y_exact), its fp32
value before rounding lay in the other value's rounding interval, so the kernel's accumulation
error was at least the distance from y_exact to that interval. The largest such distance over E is
a measured lower bound of (actual accumulation error) / E; the model requires it to be <= 1.
"""
import torch

F16_ACC_EPS = 2.0 ** -16
ACT_REL = 2.0 ** -18
U32 = 2.0 ** -24
BF16_HALF_ULP_REL = 2.0 ** -8


def scale_granule(avg):
    """Column granule of the transposed activation-scale layout for avg = T*K // E_total."""
    buckets = ((8, 8), (16, 16), (32, 32), (48, 48), (64, 64), (96, 48), (128, 32), (144, 48))
    for top, gran in buckets:
        if avg <= top:
            return gran
    return 64


def round_sig(v, bits):
    """Round fp64 `v` to `bits` significant bits, half to even (bf16: 8). Exact for normal values."""
    v = v.double()
    e = torch.floor(torch.log2(v.abs().clamp_min(1e-300)))
    q = torch.exp2(e - (bits - 1))
    return torch.where(v == 0, v, torch.round(v / q) * q)


def e4m3_ordinal(codes):
    """Monotonic integer of e4m3 codes: neighbouring values differ by 1. 0x7F / 0xFF are NaN and
    would map next to +-448: callers reject them first."""
    b = codes.view(torch.uint8).to(torch.int32)
    mag = b & 0x7F
    return torch.where(b >= 0x80, -mag, mag)


# ------------------------------------------------------------------------------------------------
# route
# ------------------------------------------------------------------------------------------------
def route(topk_ids, num_expert_local, rank_ep, num_expert_total):
    """Exact routing: dict(counts, cu, topk_pos, src_token [rows], expert_of_row [rows],
    col_of_row [rows] (column in the scale layout), pad_base, granule)."""
    T, K = topk_ids.shape
    ids = topk_ids.reshape(-1).long() - rank_ep * num_expert_local
    local = (ids >= 0) & (ids < num_expert_local)
    counts = torch.bincount(ids[local], minlength=num_expert_local).to(torch.int32)
    cu = torch.zeros(num_expert_local + 1, dtype=torch.int32)
    cu[1:] = torch.cumsum(counts, 0)
    gran = scale_granule(T * K // num_expert_total)
    padded = (counts + gran - 1) // gran * gran
    pad_base = torch.zeros(num_expert_local, dtype=torch.int64)
    pad_base[1:] = torch.cumsum(padded, 0)[:-1]
    flat = torch.arange(T * K)
    order = torch.sort(ids[local] * (T * K) + flat[local]).indices  # expert-major, then (t, k)
    slots = flat[local][order]
    rows = slots.numel()
    topk_pos = torch.full((T * K,), -1, dtype=torch.int32)
    topk_pos[slots] = torch.arange(rows, dtype=torch.int32)
    expert_of_row = ids[slots]
    j = torch.arange(rows) - cu[:-1].long()[expert_of_row]
    return dict(counts=counts, cu=cu, topk_pos=topk_pos.view(T, K), src_token=slots // K,
                expert_of_row=expert_of_row, col_of_row=pad_base[expert_of_row] + j,
                local_index=j, pad_base=pad_base, granule=gran)


def scale_layout(x_scale, r, num_padded):
    """The activation-scale layout the route kernel writes; unwritten columns are NaN."""
    out = torch.full((x_scale.size(1), num_padded), float("nan"))
    out[:, r["col_of_row"]] = x_scale[r["src_token"]].t().float()
    return out


def check_route(r, x, x_scale, got):
    """`got`: the kernel's counts, cu_counts, topk_pos, gate_up_input, gate_up_input_scale (CPU)."""
    assert torch.equal(got["counts"], r["counts"]), "route: counts differ"
    assert torch.equal(got["cu_counts"], r["cu"]), "route: cu_counts differ"
    assert torch.equal(got["topk_pos"], r["topk_pos"]), "route: topk_pos differ"
    rows = r["src_token"].numel()
    want = x.view(torch.uint8)[r["src_token"]]
    assert torch.equal(got["gate_up_input"].view(torch.uint8)[:rows], want), "route: gathered rows differ"
    lay = got["gate_up_input_scale"][:, r["col_of_row"]]
    want = x_scale[r["src_token"]].t().float()
    bad = (lay != want).any(0)
    assert not bad.any(), (f"route: activation-scale layout wrong for {int(bad.sum())} rows, first row "
                           f"{int(bad.nonzero()[0])} (granule {r['granule']})")


# ------------------------------------------------------------------------------------------------
# GEMM with its error bound
# ------------------------------------------------------------------------------------------------
def _gemm_rows(a, w, a_scale_cols, w_scale):
    """a [nr, Kdim] codes, w [N, Kdim] codes, a_scale_cols [KB, nr] f32, w_scale [N/128, KBpad] f32.
    Returns (v_exact [nr, N] fp64, E [nr, N] fp64) per the module docstring."""
    nr, kdim = a.shape
    n = w.size(0)
    kb = kdim // 128
    A = a.double().view(nr, kb, 128)
    W = w.double().view(n, kb, 128)
    P = torch.einsum("rbk,nbk->rnb", A, W)
    S = torch.einsum("rbk,nbk->rnb", A.abs(), W.abs())
    ws = w_scale[:, :kb].float().repeat_interleave(128, dim=0)  # [N, KB]
    f = (a_scale_cols.float().t()[:, None, :] * ws[None]).double()  # fl32(xs * ws) [nr, N, KB]
    fP = f * P
    v = fP.sum(-1)
    E = (f.abs() * S).sum(-1) * F16_ACC_EPS + (kb + 1) * U32 * fP.abs().sum(-1)
    return v, E


def rows_to_check(r, seed=0, n_random=4, tile_m=64):
    """Per expert: first and last rows, both sides of every 64-row tile boundary and of every scale
    granule boundary, and a seeded random sample. Returns global row indices (sorted)."""
    g = torch.Generator().manual_seed(seed)
    gran = r["granule"]
    out = []
    for e, n in enumerate(r["counts"].tolist()):
        if n == 0:
            continue
        js = {0, n - 1}
        for step in (tile_m, gran):
            for b in range(step, n, step):
                js.update((b - 1, b))
        js.update(torch.randint(0, n, (n_random,), generator=g).tolist())
        base = int(r["cu"][e])
        out.extend(base + j for j in js)
    return torch.tensor(sorted(out), dtype=torch.long)


def _per_expert(r, rows):
    ex = r["expert_of_row"][rows]
    for e in torch.unique(ex).tolist():
        yield e, rows[ex == e]


# ------------------------------------------------------------------------------------------------
# Gate-Up + fused activation
# ------------------------------------------------------------------------------------------------
def _silu_mul_f32(g, u):
    g32, u32 = g.float(), u.float()
    return (g32 / (1.0 + torch.exp(-g32))) * u32


def _e4m3_sat(v):
    return v.clamp(-448.0, 448.0).to(torch.float8_e4m3fn)


def gateup_emulate(gathered, xs_layout, r, guw, guws, rows):
    """Codes and block scales the epilogue would write for `rows`, from exact GEMM values
    (used to test the checker itself). Returns (codes [nr, I] e4m3, scales [I/128, nr] f32)."""
    inter = guw.size(1) // 2
    codes = torch.empty((rows.numel(), inter), dtype=torch.float8_e4m3fn)
    scales = torch.empty((inter // 128, rows.numel()))
    pos = {int(q): i for i, q in enumerate(rows)}
    for e, rr in _per_expert(r, rows):
        v, _ = _gemm_rows(gathered[rr], guw[e], xs_layout[:, r["col_of_row"][rr]], guws[e])
        a = _silu_mul_f32(round_sig(v[:, :inter], 8), round_sig(v[:, inter:], 8))
        blk = a.view(len(rr), inter // 128, 128)
        sc = blk.abs().amax(-1) / 448.0
        inv = 1.0 / (sc + 1e-8)
        idx = [pos[int(q)] for q in rr]
        codes[idx] = _e4m3_sat(blk * inv[..., None]).view(len(rr), inter)
        scales[:, idx] = sc.t()
    return codes, scales


def check_gateup(gathered, xs_layout, r, guw, guws, rows, codes, scale_layout_k):
    """`codes` [rows_total, I] e4m3 (the kernel's down_input), `scale_layout_k` [I/128, num_padded]
    (the kernel's down_input_scale). Returns stats; raises on a wrong scale, a code off by more than
    one step, or an unexplained one-step flip."""
    inter = guw.size(1) // 2
    nb = inter // 128
    flips = explained = 0
    worst_scale = 0.0
    for e, rr in _per_expert(r, rows):
        v, E = _gemm_rows(gathered[rr], guw[e], xs_layout[:, r["col_of_row"][rr]], guws[e])
        gv, uv = v[:, :inter], v[:, inter:]
        ge, ue = E[:, :inter], E[:, inter:]
        a = _silu_mul_f32(round_sig(gv, 8), round_sig(uv, 8)).view(len(rr), nb, 128)
        # the block maximum the kernel can reach: every element at its smallest and largest |a| over
        # the bf16 roundings that its GEMM bound leaves open
        alts = torch.stack([_silu_mul_f32(round_sig(gv + sg * ge, 8), round_sig(uv + su * ue, 8)).abs()
                            for sg in (-1, 1) for su in (-1, 1)]).view(4, len(rr), nb, 128)
        lo = alts.min(0).values.amax(-1).double() * (1 - ACT_REL)
        hi = alts.max(0).values.amax(-1).double() * (1 + ACT_REL)
        sc_k = scale_layout_k[:, r["col_of_row"][rr]].t()  # [nr, nb]
        got_amax = sc_k.double() * 448.0
        bad = ~((got_amax >= lo) & (got_amax <= hi))
        assert not bad.any(), (f"gate-up: block scale outside the range its amax can take "
                               f"(expert {e}, {int(bad.sum())} blocks)")
        amax = a.abs().amax(-1).double()
        step = torch.exp2(torch.floor(torch.log2(amax.clamp_min(1e-30))) - 7)
        worst_scale = max(worst_scale, float(((got_amax - amax).abs() / step).max()))
        inv = 1.0 / (sc_k + 1e-8)  # f32
        va = a * inv[..., None]
        want = _e4m3_sat(va).view(len(rr), inter)
        got = codes[rr]
        nan = (got.view(torch.uint8) & 0x7F) == 0x7F  # e4m3 NaN, also the scratch sentinel
        assert not nan.any(), (f"gate-up: {int(nan.sum())} NaN codes (unwritten?) in expert {e}, "
                               f"row {int(rr[int(nan.any(1).nonzero()[0])])}")
        d = (e4m3_ordinal(got) - e4m3_ordinal(want)).abs()
        assert int(d.max()) <= 1, (f"gate-up: code off by {int(d.max())} steps (expert {e}, row "
                                   f"{int(rr[int(d.max(1).values.argmax())])})")
        m = d == 1
        if not m.any():
            continue
        flips += int(m.sum())
        amb_g = round_sig(gv - ge, 8) != round_sig(gv + ge, 8)
        amb_u = round_sig(uv - ue, 8) != round_sig(uv + ue, 8)
        vf = va.view(len(rr), inter).double()
        mid = (got.float().double() + want.float().double()) / 2
        near = (vf - mid).abs() <= ACT_REL * vf.abs()
        ok = (amb_g | amb_u | near) & m
        explained += int(ok.sum())
        unexplained = m & ~ok
        assert not unexplained.any(), (f"gate-up: {int(unexplained.sum())} unexplained one-step code "
                                       f"flips (expert {e})")
    return dict(flips=flips, explained=explained, worst_scale_steps=worst_scale)


# ------------------------------------------------------------------------------------------------
# Down
# ------------------------------------------------------------------------------------------------
def down_exact(codes, di_layout, r, dw, dws, rows):
    """fp64 Down output and bound B for `rows` (from the kernel's own codes and scale layout)."""
    H = dw.size(1)
    y = torch.empty((rows.numel(), H), dtype=torch.float64)
    B = torch.empty_like(y)
    pos = {int(q): i for i, q in enumerate(rows)}
    for e, rr in _per_expert(r, rows):
        v, E = _gemm_rows(codes[rr], dw[e], di_layout[:, r["col_of_row"][rr]], dws[e])
        idx = [pos[int(q)] for q in rr]
        y[idx] = v
        B[idx] = BF16_HALF_ULP_REL * (v.abs() + E) + E
    return y, B


def check_down(out, y, B, tag="down"):
    """`out` [nr, H] bf16 rows of the kernel's down_output. Returns worst err / B."""
    err = (out.double() - y).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / B)  # B = 0 where y = 0 exactly
    assert torch.isfinite(out.double()).all(), f"{tag}: non-finite output"
    worst = float(ratio.max())
    assert worst <= 1.0, f"{tag}: err/B {worst:.3g} at {int(ratio.argmax())}"
    return worst


def accumulation_probe(out, y, B, tag="down"):
    """Measured lower bound of (accumulation error) / E for bf16 outputs `out` with exact values `y`
    and bounds B = 2^-8 (|y| + E) + E (see the module docstring). Raises if it exceeds 1."""
    E = (B - BF16_HALF_ULP_REL * y.abs()) / (1 + BF16_HALF_ULP_REL)
    o = out.double()
    moved = (o != round_sig(y, 8)) & (o != 0)
    if not moved.any():
        return 0.0
    om, ym, em = o[moved], y[moved], E[moved]
    ex = torch.floor(torch.log2(om.abs()))
    ulp = torch.exp2(ex - 7)
    # spacing between om and its bf16 neighbour on y's side (half an ulp below a power of two)
    toward_zero = torch.sign(ym - om) != torch.sign(om)
    spacing = torch.where(toward_zero & (om.abs() == torch.exp2(ex)), ulp / 2, ulp)
    lb = ((ym - om).abs() - spacing / 2).clamp_min(0)
    ratio = torch.where(lb == 0, torch.zeros_like(lb), lb / em)
    worst = float(ratio.max())
    assert worst <= 1.0, (f"{tag}: accumulation error is at least {worst:.3g} x the model's E "
                          f"({int((ratio > 1).sum())} elements)")
    return worst


# ------------------------------------------------------------------------------------------------
# reduce
# ------------------------------------------------------------------------------------------------
def reduce_exact(down_output, topk_pos, topk_scale, shared_output=None):
    """fp64 sum_k w_k x[pos] (+ shared) and its bound, from the kernel's own bf16 Down rows."""
    T, K = topk_pos.shape
    pos = topk_pos.long()
    valid = pos >= 0
    rows = down_output.double()[pos.clamp_min(0)] * valid[..., None]
    terms = rows * topk_scale.double()[..., None]
    o = terms.sum(1)
    mag = terms.abs().sum(1)
    if shared_output is not None:
        o = o + shared_output.double()
        mag = mag + shared_output.double().abs()
    E = (K + 2) * U32 * mag
    return o, BF16_HALF_ULP_REL * (o.abs() + E) + E
