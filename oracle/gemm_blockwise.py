"""fp64 oracle of the dense blockwise FP8 GEMM (csrc/gemm_blockwise_fp8.cu) and an exact restatement
of the 1x128 activation quantiser (csrc/activation.cu blockwise_fp8_quant_kernel).

Quantiser. bf16 -> fp32 is exact; amax, amax / 448, 1 / (sc + 1e-8) and the product are single
IEEE fp32 operations and e4m3 conversion is round-to-nearest with saturation, so `quant`, which
performs them in torch fp32 in that order, is bit-exact. It is the blockwise half of
masked_act.masked_act_mul_and_blockwise_quant (the kernels share that arithmetic); that function
applies SiLU * mul first and has no entry point without it, so the few lines are restated here.

GEMM. Per output (m, n) and K block kb: P_kb = e4m3 wgmma products over four k = 32 steps from a
zeroed accumulator. Each step may err by FP8_ACC_EPS = 2^-12 of the block's magnitude S_kb = sum
|a w| (the stated model of oracle/attention_exact.py), so the block's term is 4 FP8_ACC_EPS S_kb.
Then acc = fmaf(P_kb, f_kb, acc) with f_kb = fl32(xs ws): the scale product and the FMA round once
each per block (KB + 1 roundings), and with split-K the split partials are added in fp32 (split - 1
more adds), each at most 2^-24 of sum |f P| <= sum |f| S. So
  E = (4 FP8_ACC_EPS + (KB + split) 2^-24) sum_kb |f_kb| S_kb.
moe_exact._gemm_rows (the blockwise GEMM of the FusedMoE oracle) gives the exact value v = sum f P;
called on the magnitudes (|codes|, |xs|, |ws|) it gives sum |f| S exactly, since fl32(|xs| |ws|) =
|fl32(xs ws)|. A ragged last weight-scale block is served by padding w with zero rows to whole
blocks. The bf16 output is one round-to-nearest: B = 2^-8 (|y| + E) + E. Every GPU case also runs
moe_exact.accumulation_probe, which measures whether E is adequate.

`gemm_emulate` and `quant_emulate` restate the kernels in torch fp32 and take named bugs
(GEMM_BUGS, QUANT_BUGS); tests/test_gemm_blockwise_cpu.py shows the checks pass the emulation and
catch every bug.
"""
import torch

from oracle import gemm_exact as gx
from oracle import moe_exact as ox
from oracle.attention_exact import FP8_ACC_EPS

BM, BN, BK = 128, 128, 128
BLOCK_ACC_EPS = 4 * FP8_ACC_EPS  # four k = 32 wgmma steps per K block


# ------------------------------------------------------------------------------------------------
# quantiser
# ------------------------------------------------------------------------------------------------
def _quant(v, amax_cols=128, eps=1e-8):
    n = v.size(0)
    amax = v.abs().reshape(n, -1, amax_cols).amax(-1)
    sc = amax / 448.0
    inv = 1.0 / (sc + eps) if eps else 1.0 / sc
    q = (v * inv.repeat_interleave(amax_cols, -1)).clamp(-448.0, 448.0).to(torch.float8_e4m3fn)
    return q, sc.reshape(n, -1, 128 // amax_cols)[..., 0].contiguous()


def quant(x):
    """(e4m3 [M, K], sc f32 [M, K / 128]) of bf16 x [M, K]."""
    return _quant(x.float())


QUANT_BUGS = ("inv_no_eps", "scale_wrong_row", "amax_64_columns")


def quant_emulate(x, bug=None):
    """The quantiser with an optional named bug from QUANT_BUGS."""
    v = x.float()
    if bug == "inv_no_eps":
        return _quant(v, eps=0)
    if bug == "amax_64_columns":
        return _quant(v, amax_cols=64)
    q, sc = _quant(v)
    if bug == "scale_wrong_row" and sc.size(0) > 1:
        sc = torch.roll(sc, 1, 0)
    return q, sc


def quant_mismatch(q, sc, want_q, want_sc):
    """(#codes that differ, #scales that differ), comparing bits (NaN codes compare by bits)."""
    cq = int((q.contiguous().view(torch.uint8) != want_q.contiguous().view(torch.uint8)).sum())
    cs = int((sc.contiguous().view(torch.int32) != want_sc.contiguous().view(torch.int32)).sum())
    return cq, cs


# ------------------------------------------------------------------------------------------------
# GEMM
# ------------------------------------------------------------------------------------------------
def splits(k, split):
    """[(kb0, kb1)] of every split: split s takes K blocks [KB s / split, KB (s + 1) / split)."""
    kb = k // BK
    return [(kb * s // split, kb * (s + 1) // split) for s in range(split)]


def _abs_codes(t):
    return (t.view(torch.uint8) & 0x7F).view(torch.float8_e4m3fn)


def gemm_exact(x, xs, w, ws, split, rows=None, chunk=16):
    """fp64 y, bound B and E ([nr, N]) for `rows` of x (all if None)."""
    rows = torch.arange(x.size(0)) if rows is None else rows
    n, k = w.shape
    npad = ws.size(0) * BN
    wp = torch.zeros((npad, k), dtype=torch.uint8)
    wp[:n] = w.view(torch.uint8)
    wp = wp.view(torch.float8_e4m3fn)
    wa, wsa = _abs_codes(wp), ws.abs()
    eps = BLOCK_ACC_EPS + (k // BK + split) * ox.U32
    ys, Es = [], []
    for i in range(0, rows.numel(), chunk):
        r = rows[i:i + chunk]
        xr, xsr = x[r], xs[r].t()
        v, _ = ox._gemm_rows(xr, wp, xsr, ws)
        mag, _ = ox._gemm_rows(_abs_codes(xr), wa, xsr.abs(), wsa)  # sum_kb |f_kb| S_kb
        ys.append(v[:, :n])
        Es.append(eps * mag[:, :n])
    y, E = torch.cat(ys), torch.cat(Es)
    return y, ox.BF16_HALF_ULP_REL * (y.abs() + E) + E, E


def check(out, y, B, tag="gemm_blockwise_fp8"):
    """(worst err / B, accumulation probe) of the kernel's rows `out`; raises past 1."""
    return ox.check_down(out, y, B, tag), ox.accumulation_probe(out, y, B, tag)


def rows_to_check(m, n, k, seed=0, n_random=8, small=1 << 26, tile_m=64):
    """Every row when m * n * k is small; else both sides of every `tile_m`-row boundary (64: the
    warpgroup and tile boundaries), the first and last rows and a seeded sample."""
    if m * n * k <= small:
        return torch.arange(m)
    return gx.rows_to_check(torch.tensor([m]), torch.tensor([0, m]), n, k, tile_m=tile_m, seed=seed,
                            n_random=n_random, small=0)


GEMM_BUGS = ("xs_next_kblock", "ws_next_nblock", "ws_transposed", "drop_last_kblock",
             "split_missing", "split_doubled", "ragged_n_shift", "bf16_truncate",
             "subnormal_as_normal", "xs_next_row")


def gemm_emulate(x, xs, w, ws, split, rows=None, bug=None):
    """The kernel's arithmetic in torch fp32 for `rows` (all if None), with an optional named bug
    from GEMM_BUGS. Returns [nr, N] bf16; outputs a bug leaves unwritten are NaN."""
    m, k = x.shape
    n = w.size(0)
    kb_n, nb_n = k // BK, (n + BN - 1) // BN
    rows = torch.arange(m) if rows is None else rows
    A = gx._decode_e4m3(x[rows], bug)
    W = gx._decode_e4m3(w, bug)
    srow = (rows + 1).clamp(max=m - 1) if bug == "xs_next_row" else rows
    XS = xs[srow].float()  # [nr, KB]
    nb = torch.arange(n) // BN
    if bug == "ws_next_nblock":
        nb = (nb + 1) % nb_n
    flat = ws.reshape(-1).float()
    acc_splits = []
    for kb0, kb1 in splits(k, split):
        acc = torch.zeros(rows.numel(), n)
        for kb in range(kb0, kb1):
            if bug == "drop_last_kblock" and kb == kb_n - 1:
                continue
            P = A[:, kb * BK:(kb + 1) * BK] @ W[:, kb * BK:(kb + 1) * BK].t()
            xk = (kb + 1) % kb_n if bug == "xs_next_kblock" else kb
            wi = kb * nb_n + nb if bug == "ws_transposed" else nb * kb_n + kb
            f = XS[:, xk][:, None] * flat[wi][None]
            acc = (P.double() * f.double() + acc.double()).float()  # fmaf
        acc_splits.append(acc)
    total = torch.zeros(rows.numel(), n)
    for s, acc in enumerate(acc_splits):
        if bug == "split_missing" and s == split - 1 and s > 0:
            continue
        total = total + acc
        if bug == "split_doubled" and s == split - 1 and s > 0:
            total = total + acc
    if bug == "ragged_n_shift" and n % BN:
        n0 = n - n % BN
        total[:, n0:] = torch.cat([total[:, n0 + 8:], torch.full((rows.numel(), 8), float("nan"))], 1)
    return gx._bf16_truncate(total) if bug == "bf16_truncate" else total.to(torch.bfloat16)
