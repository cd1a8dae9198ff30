"""ORACLE — test infrastructure only (never imported by the product).

Fused AllReduce + residual + RMSNorm (csrc/allreduce.cu, both kernels) in fp64, a per-element
checker derived from the kernels' arithmetic, an fp32 emulation of that arithmetic with named
bugs, and a model of the low-latency (Lamport) workspace and its `buffer_flags`.

Reference, per token row (x_r = rank r's bf16 row, eps = fp32(eps) as the kernel receives it):
  S = sum_r x_r exactly,  s = bf16(S),  r = bf16(s + residual),
  z = r / sqrt(mean(r^2) + eps),  n = bf16(z),  y = bf16(n * gamma).
The kernels round in exactly these places: the reduction accumulates in fp32 and packs once
(multimem.ld_reduce acc::f32, the P2P and Lamport sums); `add_residual` rounds s + residual to bf16
(= out_residual) and squares the rounded values; `normalise` rounds x * rstd to bf16 before the
multiply by gamma, whose product of two bf16 values is exact in fp32 and is rounded once.

Where rounding may legitimately differ (u = 2^-24, gamma_d = d u / (1 - d u); rounding to bf16 is
monotone, so an fp32 value within b of v rounds to a bf16 value between bf16(v - b) and bf16(v + b)):
  * s: the fp32 sum of W terms in any order (rank order on the P2P and Lamport paths, the switch's
    order on NVLS) is within b_s = gamma_{W-1} sum_r |x_r| of S. b_s = 0 when every partial sum is
    representable: all terms are multiples of g (the smallest bf16 ulp among them) and
    sum |x_r| <= 2^24 g. So integer-grid inputs (synth family "exact") are bit-exact on every
    transport.
  * r: fl32(s + residual) is within u |s + residual| of the sum (0 under the same grid test), and
    monotone in s: r is accepted between bf16(s_lo + residual - b) and bf16(s_hi + residual + b)
    for the extreme candidates s_lo, s_hi of s.
  * n: the kernel's z' = fl(r * rsqrtf(fl(fl(T / H) + eps))) with T its fp32 sum of squares of
    the r values it wrote. Every square passes D = 8 NVEC (fma chain per thread) + 5 (warp_sum_f32)
    + kWarps (block sum) + 1 roundings, all terms >= 0: |T' - T| <= gamma_D T. The division and the
    eps add add two roundings, rsqrtf is within 2 ulp (2^-22 relative) and the product one more:
      delta = (1 + gamma_{D+2} / 2 (1 + gamma_{D+2})) (1 + 2^-22) (1 + u) - 1.
    n is accepted between bf16(z - delta |z|) and bf16(z + delta |z|) (z from the kernel's own
    out_residual row, once that row has passed), and y must be bf16(n * gamma) for one of them.
Every other element must match bit for bit; +0 and -0 compare equal (the Lamport kernel turns
a (+0, -0) pair into (+0, +0): 0x80000000 means "not yet written"). Inputs must keep H max^2
below the fp32 range and r^2 above its normal range, which synth.allreduce does.
"""
import numpy as np
import torch

U = 2.0 ** -24
RSQRT_REL = 2.0 ** -22

# block shapes of dispatch_row_kernel (HT) and dispatch_row_kernel_wide (LL): (max vectors, NVEC, THREADS)
HT_TABLE = ((32, 1, 32), (64, 1, 64), (128, 1, 128), (256, 1, 256), (512, 2, 256), (1024, 4, 256),
            (2048, 8, 256), (4096, 4, 1024))
LL_TABLE = ((32, 1, 32), (64, 1, 64), (128, 1, 128), (256, 1, 256), (512, 1, 512), (1024, 1, 1024),
            (2048, 2, 1024), (4096, 4, 1024))


def shape_of(hidden, kernel):
    """(NVEC, THREADS) the dispatcher of `kernel` ("ht" / "ll") picks for `hidden`."""
    nv = hidden // 8
    for lim, nvec, threads in HT_TABLE if kernel == "ht" else LL_TABLE:
        if nv <= lim:
            return nvec, threads
    raise ValueError(hidden)


def gamma(d):
    return d * U / (1 - d * U)


def norm_delta(nvec, threads):
    d = 8 * nvec + 5 + threads // 32 + 1 + 2
    g = gamma(d)
    return (1 + g / 2 * (1 + g)) * (1 + RSQRT_REL) * (1 + U) - 1


# ---- bf16 helpers ---------------------------------------------------------------------------------
def f64(t):
    """bf16 / fp32 torch tensor or numpy array -> float64 numpy (exact)."""
    if isinstance(t, torch.Tensor):
        return t.detach().cpu().float().numpy().astype(np.float64)
    return np.asarray(t, dtype=np.float64)


def rn_bf16(v):
    """Round float64 values to the nearest bf16 (ties to even), once. Finite inputs only."""
    v = np.ascontiguousarray(v, dtype=np.float64)
    b = torch.from_numpy(v).view(torch.int64)
    # ties to even on the top 8 significand bits of the fp64 pattern
    out = ((b + ((1 << 44) - 1) + ((b >> 45) & 1)) & -(1 << 45)).view(torch.float64).numpy()
    tiny = np.abs(v) < 2.0 ** -126  # bf16 subnormals: a fixed quantum of 2^-133
    if tiny.any():
        q = 2.0 ** -133
        out = np.where(tiny, np.rint(v / q) * q, out)
    return out


def to_bf16(v):
    return torch.from_numpy(np.ascontiguousarray(rn_bf16(v)).astype(np.float32)).to(torch.bfloat16)


def _ulp_floor(v):
    """Smallest bf16 ulp a nonzero value v can carry (its last significand bit); inf for 0."""
    v = np.ascontiguousarray(v, dtype=np.float64)
    e = (torch.from_numpy(v).view(torch.int64) >> 52) & 0x7FF
    u = (torch.clamp(e - 7, min=1023 - 133) << 52).view(torch.float64).numpy()
    return np.where(v == 0, np.inf, u)


def sum_bound(terms):
    """Bound on |fp32 sum (any order) - exact sum| over axis 0 of `terms`, per element."""
    n = terms.shape[0]
    a = np.abs(terms).sum(0)
    g = _ulp_floor(terms).min(0)
    exact = a <= np.ldexp(g, 24)
    return np.where(exact, 0.0, gamma(max(n - 1, 0)) * a)


# ---- reference and checker ------------------------------------------------------------------------
def reference(xs, residual, weight, eps):
    """(out_residual, out) of the exact reference as float64 arrays [T, H]."""
    X = np.stack([f64(x) for x in xs])
    s = rn_bf16(X.sum(0))
    r = rn_bf16(s + f64(residual))
    return r, _normalise(r, f64(weight), eps)


def _rstd(r, eps):
    return 1.0 / np.sqrt((r * r).mean(-1, keepdims=True) + float(np.float32(eps)))


def _normalise(r, w, eps):
    return rn_bf16(rn_bf16(r * _rstd(r, eps)) * w)


def check(out_res, out, xs, residual, weight, eps, kernel="ht", hidden=None):
    """Grade one call. out_res / out: the kernel's [T, H] outputs (NaN where not written).
    out_res = None grades rows another rank normalised (the high-throughput broadcast), whose
    out_residual this rank never sees: a row whose r is unambiguous is graded as if the owner had
    written the exact r; in a row where some r may take either neighbour, n is accepted anywhere
    between the extremes of r * rstd over every admissible r of the row, widened by delta.
    Returns dict(ok, written, worst_res, worst_out, amb_res, amb_out, bad_res, bad_out, bad_mask,
    amb_mask, widened_rows): worst_* in bf16 ulps from the exact reference; amb_* = elements where
    the accepted set holds two values; bad_* = elements outside it."""
    X = np.stack([f64(x) for x in xs])
    r_exact, y_exact = reference(xs, residual, weight, eps)
    res, w, o_y = f64(residual), f64(weight), f64(out)
    o_r = r_exact if out_res is None else f64(out_res)
    H = hidden or X.shape[-1]
    nvec, threads = shape_of(H, kernel)
    S = X.sum(0)
    bs = sum_bound(X)
    # r = bf16(fl32(s + residual)) is monotone in s: its range is spanned by the extreme s
    s_lo, s_hi = rn_bf16(S - bs), rn_bf16(S + bs)
    r_lo = rn_bf16(s_lo + res - sum_bound(np.stack([s_lo, res])))
    r_hi = rn_bf16(s_hi + res + sum_bound(np.stack([s_hi, res])))
    ok_r = (o_r >= r_lo) & (o_r <= r_hi)
    amb_r = r_lo != r_hi
    # the norm of the kernel's own rows where they passed, of the exact rows elsewhere
    row_ok = ok_r.all(-1, keepdims=True)
    r_used = np.where(row_ok, o_r, r_exact)
    z = r_used * _rstd(r_used, eps)
    d = norm_delta(nvec, threads) * np.abs(z)
    n_lo, n_hi = rn_bf16(z - d), rn_bf16(z + d)
    y_lo, y_hi = rn_bf16(n_lo * w), rn_bf16(n_hi * w)
    ok_y = (o_y == y_lo) | (o_y == y_hi)
    amb_y = y_lo != y_hi
    widen = amb_r.any(-1) if out_res is None else np.zeros(len(o_y), bool)
    if widen.any():
        lo, hi, wk = r_lo[widen], r_hi[widen], w
        sq_lo = np.where((lo <= 0) & (hi >= 0), 0.0, np.minimum(lo * lo, hi * hi))
        sq_hi = np.maximum(lo * lo, hi * hi)
        e32 = float(np.float32(eps))
        rs = [1.0 / np.sqrt(sq.mean(-1, keepdims=True) + e32) for sq in (sq_lo, sq_hi)]
        zc = np.stack([r * q for r in (lo, hi) for q in rs])
        z_lo, z_hi = zc.min(0), zc.max(0)
        dz = norm_delta(nvec, threads) * np.maximum(np.abs(z_lo), np.abs(z_hi))
        ya, yb = rn_bf16(rn_bf16(z_lo - dz) * wk), rn_bf16(rn_bf16(z_hi + dz) * wk)
        ow = o_y[widen]
        ok_y[widen] = (ow >= np.minimum(ya, yb)) & (ow <= np.maximum(ya, yb))
        amb_y[widen] = ya != yb
    written = bool(np.isfinite(o_r).all() and np.isfinite(o_y).all())

    def ulps(o, ref):
        e = np.abs(o - ref) / _ulp_floor(np.where(ref == 0, 2.0 ** -133, ref))
        return float(np.nan_to_num(e, nan=np.inf).max()) if e.size else 0.0

    bad_r, bad_y = ~ok_r, ~ok_y
    return dict(ok=written and not bad_r.any() and not bad_y.any(), written=written,
                worst_res=ulps(o_r, r_exact), worst_out=ulps(o_y, y_exact),
                amb_res=int(amb_r.sum()), amb_out=int(amb_y.sum()),
                bad_res=int(bad_r.sum()), bad_out=int(bad_y.sum()),
                bad_mask=bad_r | bad_y, amb_mask=amb_r | amb_y, widened_rows=int(widen.sum()))


def summary(tag, res):
    return (f"EXACT {tag} ok={res['ok']} written={res['written']} worst_ulp(res,out)="
            f"{res['worst_res']:.0f},{res['worst_out']:.0f} ambiguous(res,out)={res['amb_res']},"
            f"{res['amb_out']} bad(res,out)={res['bad_res']},{res['bad_out']}")


# ---- fp32 emulation of the kernels ----------------------------------------------------------------
MUTANTS = ("bf16_sum", "unrounded_norm", "no_eps", "gamma_first", "padded_width", "row_shift",
           "drop_rank")


def _f32(v):
    return np.asarray(v, dtype=np.float32)


def emulate(xs, residual, weight, eps, kernel="ht", mutant=None):
    """(out_residual, out) as float64 arrays, computed in fp32 in the kernel's order: rank-order
    fp32 sum (as the P2P and Lamport paths), add_residual, the per-thread fma chain, the xor
    butterfly, the block sum, rsqrt, normalise. `mutant` names a bug (MUTANTS)."""
    X = [f64(x) for x in xs]
    if mutant == "drop_rank" and len(X) > 1:
        X = X[:-1]
    T, H = X[0].shape
    nvec, threads = shape_of(H, kernel)
    if mutant == "bf16_sum":
        acc = np.zeros((T, H))
        for x in X:
            acc = rn_bf16(acc + x)
        s = acc
    else:
        acc = _f32(np.zeros((T, H)))
        for x in X:
            acc = acc + _f32(x)
        s = rn_bf16(acc.astype(np.float64))
    unrounded = _f32(s) + _f32(f64(residual))
    r = rn_bf16(unrounded.astype(np.float64))
    a = unrounded.astype(np.float64) if mutant == "unrounded_norm" else r
    # per thread: vectors v = tid + j THREADS, 8 elements each, sq = fma(a, a, sq) in order
    pad = np.zeros((T, nvec * threads * 8))
    pad[:, :H] = a
    pv = pad.reshape(T, nvec, threads, 8)
    sq = _f32(np.zeros((T, threads)))
    for j in range(nvec):
        for i in range(8):
            e = pv[:, j, :, i]
            sq = _f32(e * e + sq.astype(np.float64))  # fma: one rounding
    w_ = sq.reshape(T, threads // 32, 32)
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        w_ = w_ + w_[:, :, lane ^ o]
    tot = _f32(np.zeros(T))
    for k in range(threads // 32):
        tot = tot + w_[:, k, 0]
    width = nvec * threads * 8 if mutant == "padded_width" else H
    e32 = np.float32(0.0 if mutant == "no_eps" else eps)
    m = _f32(_f32(tot / np.float32(width)) + e32)
    with np.errstate(divide="ignore", invalid="ignore"):  # no_eps on an all-zero row
        rstd = _f32(1.0 / np.sqrt(m.astype(np.float64)))[:, None]
    w = f64(weight)
    with np.errstate(invalid="ignore"):
        z = _f32(_f32(a) * rstd).astype(np.float64)
    if mutant == "gamma_first":
        y = rn_bf16(z * w)
    else:
        y = rn_bf16(rn_bf16(z) * w)
    if mutant == "row_shift" and T > 1:
        r, y = np.roll(r, 1, 0), np.roll(y, 1, 0)
    return r, y


def emulate_sum(xs):
    """Rank-order fp32 sum packed to bf16: what an owner broadcasts on the two-shot path."""
    acc = _f32(np.zeros(f64(xs[0]).shape))
    for x in xs:
        acc = acc + _f32(f64(x))
    return rn_bf16(acc.astype(np.float64))


def old_check(out_res, out, ref_res, ref_out):
    """The parity check the multi-GPU tests used before: allclose at atol = rtol = 0.1."""
    c = lambda a, b: torch.allclose(torch.as_tensor(a).float(), torch.as_tensor(b).float(),  # noqa: E731
                                    atol=0.1, rtol=0.1)
    return c(out_res, ref_res) and c(out, ref_out)


# ---- low-latency workspace model ------------------------------------------------------------------
NEG_ZERO_WORD = 0x80000000
ONE_SHOT_MAX_BYTES = 2 << 20


def ll_protocol(T, W, H, buf_bytes, protocol):
    """(one_shot, bytes recorded in buffer_flags[4]) for a call (allreduce.cu, kernel prologue)."""
    row = 2 * H
    tpr = (T + W - 1) // W
    one = T * W * row
    two = tpr * W * row + T * row
    one_shot = protocol == 0 and one <= buf_bytes and one <= ONE_SHOT_MAX_BYTES
    return one_shot, one if one_shot else two


def ll_flags_after(flags, T, W, H, protocol):
    """buffer_flags after one call, and the byte range of buffer `dirty` that call clears."""
    f = list(flags)
    cur, dirty, buf_bytes, dirty_bytes = f[0] % 3, f[1] % 3, f[2], f[4]
    clear = (dirty, 0 if dirty == cur else (min(dirty_bytes, buf_bytes) + 15) // 16 * 16)
    _, used = ll_protocol(T, W, H, buf_bytes, protocol)
    f[8], f[1], f[4], f[0] = 0, cur, used, (cur + 1) % 3
    return f, clear


def ll_rows(T, W, H, one_shot):
    """Byte offsets (within one buffer) of the rows of the layout:
    slot(t, r) = where rank r's row of token t lands on its destination rank,
    dest(t, r) = the rank that receives it (None = every rank), stage1(t) = the reduced row of t."""
    row = 2 * H
    tpr = (T + W - 1) // W
    if one_shot:
        return (lambda t, r: (t * W + r) * row), (lambda t, r: None), None
    return ((lambda t, r: ((t // W) * W + r) * row), (lambda t, r: t % W),
            (lambda t: tpr * W * row + t * row))


def scrub(rows_bf16):
    """A kernel-side store of bf16 rows: every 32-bit word equal to 0x80000000 becomes 0."""
    w = rows_bf16.contiguous().view(torch.int32).clone()
    w[w == -2147483648] = 0
    return w.view(torch.bfloat16)


def ll_peer_images(T, W, H, rank, one_shot, x_rank, sums, buf_words, peers=None):
    """What rank `rank`'s launch stores into the current buffer of each rank in `peers` (default:
    every p != rank), as int32 word arrays with the sentinel where it stores nothing.
    x_rank: [T, H] bf16, sums: [T, H] bf16 reduced rows (two-shot)."""
    slot, dest, stage1 = ll_rows(T, W, H, one_shot)
    row_w = H // 2
    peers = [p for p in range(W) if p != rank] if peers is None else peers
    imgs = {p: np.full(buf_words, -2147483648, np.int32) for p in peers}
    xw = scrub(x_rank).view(torch.int32).reshape(T, row_w).numpy()
    sw = None if sums is None else scrub(sums).view(torch.int32).reshape(T, row_w).numpy()
    for t in range(T):
        d = dest(t, rank)
        for p in imgs:
            if d is None or d == p:
                o = slot(t, rank) // 4
                imgs[p][o:o + row_w] = xw[t]
            if stage1 is not None and t % W == rank:
                o = stage1(t) // 4
                imgs[p][o:o + row_w] = sw[t]
    return imgs


def ll_prefill(T, W, H, rank, one_shot, xs, sums, buf_words, poison_word):
    """The launching rank's current buffer before a simulated-peer launch: the peers' rows where
    the layout puts them (scrubbed, as a peer's kernel stores them), the owners' reduced rows of
    tokens this rank does not own, and a finite poison word everywhere else, so that no 16-byte
    vector holds the sentinel and no wait can spin."""
    slot, dest, stage1 = ll_rows(T, W, H, one_shot)
    row_w = H // 2
    img = np.full(buf_words, poison_word, np.int32)
    xw = [scrub(x).view(torch.int32).reshape(T, row_w).numpy() for x in xs]
    sw = None if sums is None else scrub(sums).view(torch.int32).reshape(T, row_w).numpy()
    for t in range(T):
        for r in range(W):
            if r == rank:
                continue
            d = dest(t, r)
            if d is None or d == rank:
                o = slot(t, r) // 4
                img[o:o + row_w] = xw[r][t]
        if stage1 is not None and t % W != rank:
            o = stage1(t) // 4
            img[o:o + row_w] = sw[t]
    return img


def ceil_div(a, b):
    return -(-a // b)
