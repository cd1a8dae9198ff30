"""ORACLE — test infrastructure only (never imported by the product).

Fused RMSNorm -> FP8 (hpc.fused_rmsnorm_with_scale) in fp64, with a per-element bound on the
kernel's fp32 output and an e4m3 check that admits a code flip only where it is explained.

The reference's ground truth (reference tests/test_normalization.py:13-28,
`reference_torch_rmsnorm_with_scale` / `reference_torch_rmsnorm`) is torch fp32; it pins this
oracle through tests/golden/norm_*.npz (tests/golden/make_golden_norm_act.py).

Bound on the fp32 output y = (x * w) * r, r = rsqrtf(ss / H + eps), derived from the kernel's
arithmetic (csrc/normalization.cu); u = 2^-24, gamma_d = d u / (1 - d u):

  * x and w are bf16, exact in fp32, and x * w (8 + 8 significant bits) is exact.
  * ss: each thread fma-accumulates its 8 * kIter squares in order, a 5-level warp butterfly adds
    the lanes and kWpr - 1 further adds join the warps of a row, so every square passes at most
    d = 8 kIter + 5 + (kWpr - 1) roundings: |ss^ - ss| <= gamma_d ss.
  * m^ = fl(fl(ss^ / H) + eps) with eps the fp32 value passed: two more roundings, so
    |m^ / m - 1| <= e_m = (1 + gamma_d)(1 + u)^2 - 1 (the eps term carries less error than ss / H).
  * rsqrtf is within 2 ulp, i.e. a relative 2^-22, of m^^-1/2, and m^^-1/2 is within
    (1 - e_m)^-1/2 - 1 of m^-1/2: e_r = (1 + 2^-22)(1 - e_m)^-1/2 - 1.
  * Two fp32 products, x * w (exact here, counted anyway) and * r: e_y = (1 + e_r)(1 + u)^2 - 1.
  => |y^ - y| <= e_y |y| + 2^-149 (the smallest fp32 subnormal, for outputs that underflow).

For the e4m3 codes the kernel forms p = fl(y^ * fl(1 / s)), two more roundings:
|p - y / s| <= b = ((1 + e_y)(1 + u)^2 - 1) |y / s| + 2^-149 |1 / s|. cvt.rn.satfinite is monotone,
so the kernel's code must lie between the codes of y / s - b and y / s + b; when those differ the
fp64 value sits within the bound of a rounding boundary and a flip to either is "explained".
"""
import numpy as np

U = 2.0 ** -24
RSQRT_REL = 2.0 ** -22
TINY = 2.0 ** -149
WARPS = 8  # warps per CTA of the kernel


def layout(hidden):
    """(warps per row, 16-byte vectors per thread) the launcher picks for `hidden`."""
    nvec = hidden // 8
    wpr = 1
    while wpr < WARPS and nvec > wpr * 32 * 4:
        wpr *= 2
    return wpr, -(-nvec // (wpr * 32))


def _gamma(d):
    return d * U / (1 - d * U)


def rel_bound(hidden):
    """e_y of the module docstring: relative bound on the kernel's fp32 output."""
    wpr, it = layout(hidden)
    e_m = (1 + _gamma(8 * it + 5 + wpr - 1)) * (1 + U) ** 2 - 1
    e_r = (1 + RSQRT_REL) * (1 - e_m) ** -0.5 - 1
    return (1 + e_r) * (1 + U) ** 2 - 1


def _f64(t):
    import torch

    return t.detach().cpu().to(torch.float64).numpy() if isinstance(t, torch.Tensor) else np.asarray(t, np.float64)


def rmsnorm(x, w, eps):
    """fp64 y = x * w / sqrt(mean(x^2) + eps), eps taken as the fp32 value the kernel receives."""
    x = _f64(x)
    w = _f64(w).reshape(-1)
    x = x.reshape(-1, x.shape[-1])
    m = (x * x).sum(-1, keepdims=True) / x.shape[-1] + float(np.float32(eps))
    return x * w / np.sqrt(m)


def y_bound(y):
    """Per-element bound on |kernel fp32 output - y| for y = rmsnorm(...)."""
    return rel_bound(y.shape[-1]) * np.abs(y) + TINY


# ---- e4m3 (fn: no inf, 0x7F = NaN) round-to-nearest-even with saturation to +-448 ----------------
def _e4m3_table():
    vals = np.zeros(127)
    for c in range(127):
        e, m = c >> 3, c & 7
        vals[c] = (m / 8) * 2.0 ** -6 if e == 0 else (1 + m / 8) * 2.0 ** (e - 7)
    return vals


E4M3 = _e4m3_table()


def e4m3_code(v):
    """Codes (uint8) of cvt.rn.satfinite.e4m3 for float64 values (no NaN inputs)."""
    v = np.asarray(v, np.float64)
    a = np.minimum(np.abs(v), 448.0)
    hi = np.clip(np.searchsorted(E4M3, a, side="left"), 1, 126)
    lo = hi - 1
    dl, dh = a - E4M3[lo], E4M3[hi] - a
    pick_hi = (dh < dl) | ((dh == dl) & (hi % 2 == 0))
    mag = np.where(pick_hi, hi, lo)
    mag = np.where(a >= E4M3[126], 126, mag)
    return (mag | np.where(v < 0, 0x80, 0)).astype(np.uint8)


def _ordinal(code):
    c = np.asarray(code).astype(np.int32)
    return np.where(c & 0x80, -(c & 0x7F), c & 0x7F)


def check_codes(codes, y, scale, rel=None):
    """Kernel e4m3 codes against fp64 y / scale. Returns (unexplained, explained_flips): a code
    that differs from the fp64 value's rounding counts as explained only when a rounding boundary
    lies within the bound of that value."""
    rel = rel_bound(y.shape[-1]) if rel is None else rel
    s = float(np.float32(scale))
    v = y / s
    b = ((1 + rel) * (1 + U) ** 2 - 1) * np.abs(v) + TINY / abs(s)
    return check_codes_within(codes, v, b)


def check_codes_within(codes, v, b):
    """Kernel e4m3 codes against fp64 values v whose kernel-side fp32 value is within b of v.
    Returns (unexplained, explained_flips) as check_codes does."""
    codes = np.asarray(codes).astype(np.uint8)
    lo, hi = _ordinal(e4m3_code(v - b)), _ordinal(e4m3_code(v + b))
    k = _ordinal(codes)
    ok = (k >= lo) & (k <= hi)
    flips = ok & (k != _ordinal(e4m3_code(v)))
    return int((~ok).sum()), int(flips.sum())


def check(out, x, w, eps, scale, is_moe):
    """The GPU test's whole check of one call: out = q0 or (y32, q0, q1) as numpy / torch.
    Returns a dict of failure counts (all must be 0) and explained flips."""
    y = rmsnorm(x, w, eps)
    sc = _f64(scale).reshape(-1)
    res = {}
    if is_moe:
        y32, q0, q1 = out
        y32 = _f64(y32).reshape(y.shape)
        res["fp32"] = int((~(np.abs(y32 - y) <= y_bound(y))).sum())
        res["q1"], res["flips_q1"] = check_codes(_u8(q1).reshape(y.shape), y, sc[1])
    else:
        q0 = out
    res["q0"], res["flips_q0"] = check_codes(_u8(q0).reshape(y.shape), y, sc[0])
    return res


def _u8(t):
    import torch

    if isinstance(t, torch.Tensor):
        return t.detach().cpu().contiguous().view(torch.uint8).numpy()
    return np.asarray(t).astype(np.uint8)


def failed(res):
    return any(v for k, v in res.items() if not k.startswith("flips"))
