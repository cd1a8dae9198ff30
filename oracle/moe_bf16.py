"""Stage-by-stage fp64 oracle of the bf16 FusedMoE pipeline (csrc/fuse_moe.cu
hpc_fuse_moe_bf16_async, csrc/group_gemm_bf16.cu), in the manner of oracle/moe_exact.py, whose
route / check_route / rows_to_check / reduce_exact / check_down / accumulation_probe it reuses.

Each stage is computed from the kernel's own input to that stage (the rows the route kernel
gathered, the bf16 activation the Gate-Up epilogue wrote, the bf16 rows the Down GEMM wrote), so no
stage inherits an earlier stage's rounding.

route (exact): as moe_exact.route; the bf16 rows are compared bytewise, and `tiles` counts each
expert's 128-row m-tiles of the bf16 GEMM.

GEMM arithmetic (both GEMMs). bf16 x bf16 products are exact in fp32. The tensor core adds them
into an fp32 accumulator, chained over the whole K (one m64n256k16 wgmma per 16 K values). How
Hopper's tensor cores add inside a wgmma is not documented, so the bound is a stated model, not a
derivation: every one of the K additions is an fp32 add that may truncate, i.e. errs by at most
2^-23 of a partial sum, and every partial sum is at most S = sum_k |a_k w_k|. So the pre-rounding
value v has |v - v_exact| <= E = K 2^-23 S. `accumulation_probe` measures a lower bound of
(actual error) / E from the outputs; the model requires it to be <= 1.

Gate-Up epilogue: g, u = bf16_rn(v) for the gate and up columns; a = bf16_rn(silu(g) * u) with
silu = __fdividef(x, 1 + __expf(-x)) and the product in fp32. A down_input element may differ from
the oracle's bf16_rn(a) only where that is explained:
  (i)  g or u lies within E of a bf16 rounding boundary (bf16_rn(v - E) != bf16_rn(v + E)), or
  (ii) a lies within ACT_REL of the boundary between the two bf16 values; ACT_REL = 2^-18 covers
       __expf, __fdividef and the product (moe_exact.ACT_REL).
Away from zero that is one bf16 step; check_gateup bounds it exactly by the range a can take.

Down (bf16 output): |out - y_exact| <= B = 2^-8 (|y_exact| + E) + E (half an ulp of 8 significant
bits plus the accumulation bound), checked with moe_exact.check_down.

reduce: moe_exact.reduce_exact, unchanged (the same kernel reads the bf16 Down rows).
"""
import torch

from oracle import moe_exact as ox

ACC_ULP = 2.0 ** -23
ACT_REL = ox.ACT_REL
TILE_M = 128  # rows of a bf16 GEMM tile
SILU_ARGMIN = -1.2784645  # silu's minimum: x = -1 - W(1/e)
SILU_MIN = -0.27846454


def route(topk_ids, num_expert_local, rank_ep, num_expert_total):
    """moe_exact.route (the routing is the FP8 pipeline's, unchanged)."""
    return ox.route(topk_ids, num_expert_local, rank_ep, num_expert_total)


def check_route(r, x, got):
    """`got`: the kernel's counts, cu_counts, topk_pos, gate_up_input, tiles, cu_tiles (CPU).
    The rows are compared as bytes by moe_exact.check_route, given an empty activation-scale
    layout (bf16 rows carry no scales)."""
    cols = int(r["col_of_row"].max()) + 1 if r["col_of_row"].numel() else 1
    ox.check_route(r, x, torch.empty((x.size(0), 0)),
                   dict(got, gate_up_input_scale=torch.empty((0, cols))))
    tiles = (r["counts"] + TILE_M - 1) // TILE_M
    assert torch.equal(got["tiles"], tiles), "route: tiles differ"
    cu = torch.zeros_like(r["cu"])
    cu[1:] = torch.cumsum(tiles, 0)
    assert torch.equal(got["cu_tiles"], cu), "route: cu_tiles differ"


def rows_to_check(r, seed=0, n_random=4):
    """moe_exact.rows_to_check at the bf16 GEMM's 128-row tile boundaries."""
    return ox.rows_to_check(r, seed=seed, n_random=n_random, tile_m=TILE_M)


def gemm_rows(a, w):
    """a [nr, K] bf16, w [N, K] bf16 -> (v_exact [nr, N] fp64, E [nr, N] fp64)."""
    A, W = a.double(), w.double()
    v = A @ W.t()
    E = a.size(1) * ACC_ULP * (A.abs() @ W.abs().t())
    return v, E


def _per_expert(r, rows):
    ex = r["expert_of_row"][rows]
    for e in torch.unique(ex).tolist():
        yield e, rows[ex == e]


def silu_mul(g, u):
    """fp32 silu(g) * u of bf16-valued g and u (the epilogue's chain with exact exp / division)."""
    g32, u32 = g.float(), u.float()
    return (g32 / (1.0 + torch.exp(-g32))) * u32


def bf16_ordinal(v):
    """Monotonic integer of bf16 values: neighbouring values differ by 1."""
    b = v.contiguous().view(torch.int16).to(torch.int32)
    mag = b & 0x7FFF
    return torch.where(b < 0, -mag, mag)


def gateup_emulate(gathered, r, guw, rows):
    """The bf16 activation the epilogue would write for `rows`, from exact GEMM values (used to
    test the checker itself). Returns [nr, I] bf16."""
    inter = guw.size(1) // 2
    out = torch.empty((rows.numel(), inter), dtype=torch.bfloat16)
    pos = {int(q): i for i, q in enumerate(rows)}
    for e, rr in _per_expert(r, rows):
        v, _ = gemm_rows(gathered[rr], guw[e])
        a = silu_mul(ox.round_sig(v[:, :inter], 8), ox.round_sig(v[:, inter:], 8))
        out[[pos[int(q)] for q in rr]] = a.to(torch.bfloat16)
    return out


def _silu_range(lo, hi):
    """Elementwise [min, max] of fp32 silu over bf16-valued intervals [lo, hi] (silu decreases
    below its minimum at SILU_ARGMIN and increases above it)."""
    a, b = silu_mul(lo, torch.ones_like(lo)), silu_mul(hi, torch.ones_like(hi))
    mn = torch.minimum(a, b)
    inside = (lo <= SILU_ARGMIN) & (SILU_ARGMIN <= hi)
    return torch.where(inside, torch.full_like(mn, SILU_MIN), mn), torch.maximum(a, b)


def check_gateup(gathered, r, guw, rows, down_input):
    """`gathered` the kernel's gate_up_input, `down_input` its [rows_total, I] bf16 activation.
    Returns stats; raises where a value is not bf16_rn(a) and not explained.

    The explanation: g lies in [v_g - E, v_g + E], so bf16_rn(g) is one of the bf16 values from
    bf16_rn(v_g - E) to bf16_rn(v_g + E) (and likewise u); a = silu(g) * u then lies between the
    extremes of silu over that range times the extremes of u (a bilinear product takes its extremes
    at the corners), widened by ACT_REL, and the kernel's value is its bf16 rounding. Where E covers
    no bf16 boundary that range is one value up to ACT_REL, i.e. at most one bf16 step (cases (i)
    and (ii) of the module docstring); a g or u that cancels to near zero can be several of its own
    bf16 steps away, and so can a."""
    inter = guw.size(1) // 2
    flips = explained = max_steps = 0
    for e, rr in _per_expert(r, rows):
        v, E = gemm_rows(gathered[rr], guw[e])
        gv, uv = v[:, :inter], v[:, inter:]
        ge, ue = E[:, :inter], E[:, inter:]
        a = silu_mul(ox.round_sig(gv, 8), ox.round_sig(uv, 8))
        want = a.to(torch.bfloat16)
        got = down_input[rr]
        assert torch.isfinite(got.float()).all(), (f"gate-up: non-finite (unwritten?) values in expert "
                                                   f"{e}")
        m = got.view(torch.int16) != want.view(torch.int16)
        m &= (got.float() != want.float())  # +0 and -0
        if not m.any():
            continue
        flips += int(m.sum())
        s_lo, s_hi = _silu_range(ox.round_sig(gv - ge, 8).float(), ox.round_sig(gv + ge, 8).float())
        u_lo, u_hi = ox.round_sig(uv - ue, 8).float(), ox.round_sig(uv + ue, 8).float()
        corners = torch.stack([s_lo * u_lo, s_lo * u_hi, s_hi * u_lo, s_hi * u_hi]).double()
        lo, hi = corners.min(0).values, corners.max(0).values
        lo = (lo - ACT_REL * lo.abs()).float().to(torch.bfloat16).double()
        hi = (hi + ACT_REL * hi.abs()).float().to(torch.bfloat16).double()
        g64 = got.double()
        ok = (g64 >= lo) & (g64 <= hi) & m
        explained += int(ok.sum())
        d = (bf16_ordinal(got) - bf16_ordinal(want)).abs()
        max_steps = max(max_steps, int(d[m].max()))
        unexplained = m & ~ok
        assert not unexplained.any(), (
            f"gate-up: {int(unexplained.sum())} unexplained differences (expert {e}, row "
            f"{int(rr[int(unexplained.any(1).nonzero()[0])])}, up to {int(d[unexplained].max())} "
            f"bf16 steps)")
    return dict(flips=flips, explained=explained, max_steps=max_steps)


def down_exact(down_input, r, dw, rows):
    """fp64 Down output and bound B for `rows` (from the kernel's own bf16 activation)."""
    H = dw.size(1)
    y = torch.empty((rows.numel(), H), dtype=torch.float64)
    B = torch.empty_like(y)
    pos = {int(q): i for i, q in enumerate(rows)}
    for e, rr in _per_expert(r, rows):
        v, E = gemm_rows(down_input[rr], dw[e])
        idx = [pos[int(q)] for q in rr]
        y[idx] = v
        B[idx] = ox.BF16_HALF_ULP_REL * (v.abs() + E) + E
    return y, B


def group_gemm_exact(x, w, seqlens, cu_seqlens):
    """fp64 Y and bound B of group_gemm_bf16 for every row of every group; rows outside the groups
    are NaN."""
    M, N = x.size(0), w.size(1)
    y = torch.full((M, N), float("nan"), dtype=torch.float64)
    B = torch.full_like(y, float("nan"))
    for g in range(w.size(0)):
        n, r0 = int(seqlens[g]), int(cu_seqlens[g])
        if n == 0:
            continue
        v, E = gemm_rows(x[r0:r0 + n], w[g])
        y[r0:r0 + n] = v
        B[r0:r0 + n] = ox.BF16_HALF_ULP_REL * (v.abs() + E) + E
    return y, B


def reference_fp32(x, guw, dw, topk_ids, topk_scale, rank_ep, num_expert_total, shared_output=None):
    """The contract restated naively in fp32 torch (per token, per k, per expert; no routing
    tables): returns the [T, H] bf16 output."""
    T, H = x.shape
    E = guw.size(0)
    inter = guw.size(1) // 2
    y = torch.zeros((T, H), dtype=torch.float32)
    for t in range(T):
        for k in range(topk_ids.size(1)):
            e = int(topk_ids[t, k]) - rank_ep * E
            if not 0 <= e < E:
                continue
            gu = (x[t].float() @ guw[e].float().t()).to(torch.bfloat16).float()
            a = silu_mul(gu[:inter], gu[inter:]).to(torch.bfloat16).float()
            d = (a @ dw[e].float().t()).to(torch.bfloat16).float()
            y[t] += topk_scale[t, k].float() * d
    if shared_output is not None:
        y += shared_output.float()
    return y.to(torch.bfloat16)
