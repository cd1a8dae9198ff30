"""ORACLE — test infrastructure only (never imported by the product).

RoPE (NeoX halves) + QK RMSNorm + paged KV store (hpc.rope_norm_store_kv[_fp8]) in fp64, with a
per-element bound on the kernel's fp32 value derived from the arithmetic of csrc/rope.cu, the
launch predicate of that file, the cache contract, and an fp32 emulation of both kernels with
named bugs (`emulate(..., mutation=)`) that the CPU tests use to show the check catches them.

Reference values. Inputs are the bf16 qkv (exact in fp64), the fp32 cos | sin table AS GIVEN (the
kernel only reads it; no angle is recomputed), fp32 norm weights and eps = fp32(1e-6). For a
rotation pair (a, b) = (x_i, x_{i+D/2}) with c, s of the token's row:
  lower y_i = a c - b s,  upper y_{i+D/2} = b c + a s,  t_i = |a c| + |b s| (resp. |b c| + |a s|).
RMS factor r = (S / D + eps)^-1/2 with S the sum of squares of the head's D values. Policy 0: no
norm; 2: x -> x r w before the rotation; 1: y -> y r w after it.

Bound (u = 2^-24, gamma_d = d u / (1 - d u)), per element, on |kernel fp32 - y|:
  * Rotation. The kernel forms a*c -/+ b*s with two products and one add, or one product and an
    fma when nvcc contracts (-O3, --fmad=true): either way at most two roundings per term, so
    |y^ - y| <= gamma_2 t (relative to t, not to y: y can cancel).
  * Sum of squares. d128 kernel: a lane owns 4 dims and sums 4 squares, then a 5-level xor
    butterfly: every square passes at most d = 4 + 5 roundings. Generic kernel: a lane owns
    4 kCH dims (kCH 64-dim chunks per half): d = 4 kCH + 5. All terms are >= 0, so
    |S^ - S| <= gamma_d S.
  * m^ = fl(fl(S^ / D) + eps): IEEE division (no fast math) and one add, eps exact:
    e_m = (1 + e_S)(1 + u)^2 - 1 with e_S the relative error of S^.
  * rsqrtf is within 2 ulp (2^-22 relative) of m^^-1/2: e_r = (1 + 2^-22)(1 - e_m)^-1/2 - 1.
  * x * fl(r w): two products, e_a = (1 + e_r)(1 + u)^2 - 1 relative to x r w.
  Policy 0: b = gamma_2 t.
  Policy 2: e_S = gamma_d (S of the bf16 inputs, exact); the rotation then runs on values within
    e_a of A = x r w: b = ((1 + e_a)(1 + gamma_2) - 1) T, T = |A_lo c| + |A_hi s| per element.
  Policy 1: the RMS is taken over the rotated values y^, |y^_i - y_i| <= gamma_2 t_i, so
    |sum y^^2 - S| <= Delta = gamma_2 sum t_i (2 |y_i| + gamma_2 t_i) and
    e_S = (Delta / S)(1 + gamma_d) + gamma_d per head; then
    b = |r w| (gamma_2 t (1 + e_a) + e_a |y|) with y the unnormalised rotation.
  Every bound adds 2^-149 for outputs that underflow.

Outputs. A bf16 output (rn of the fp32 value, monotone) must lie between the bf16 roundings of
y - b and y + b; an e4m3 code (cvt.rn.satfinite of p = fl(y^ * mult)) between the codes of
v - b_v and v + b_v with v = y mult, b_v = |mult| (b (1 + u) + u |y|) + 2^-149
(oracle.normalization.check_codes_within). A value that differs from the rounding of the fp64
value inside those limits is an explained flip; anything else is unexplained.
  * Dynamic Q scale (quant_policy 1): the kernel writes qs = fl(max |y^| / upper_max); with
    max |y^| in [max(|y| - b), max(|y| + b)], qs must lie in that range / upper_max widened by
    one rounding. The codes are then checked with mult = fl(1 / qs) (= __frcp_rn) of the
    kernel's own qs (0 when qs is 0).
  * Static scales: mult = q_scale_inv as given for Q (quant_policy 2), fl(1 / k_scale) for K.
  * V is copied (bf16) or quantised as fl(v * fl(1 / v_scale)) (fp8): one fp32 value, so V must
    match bit for bit.

Cache contract. A call owns, in the page of every row with a position, that row's slot (all kv
heads), and when a request has rows in the call, the slots after its last token in that page,
which must be zero. Every other byte of the cache buffer -- other pages, other slots, the other
half of a combined [blocks, 2, page, Hkv, D] cache, the pages of requests with no rows -- must be
unchanged. With out_k / out_v the call writes no cache byte at all.
"""
import numpy as np

from oracle.normalization import RSQRT_REL, TINY, U, check_codes_within, e4m3_code

EPS = float(np.float32(1e-6))
FP8_MAX = 448.0
MUTATIONS = (
    "pos+1", "pos-1", "cos_sin_swapped", "rotation_sign", "gptj_pairs", "rms_bf16", "eps_dropped",
    "eps_1e-5", "rms_half_dims", "qk_norm_weights_swapped", "weight_halves_swapped",
    "policies_swapped", "upper_max_ignored", "k_times_scale", "v_with_k_scale", "tail_from_pb",
    "tail_every_page", "k_tail_head0", "dense_page_stride", "q_scale_column_row",
)
FP8_ONLY = ("upper_max_ignored", "k_times_scale", "v_with_k_scale", "q_scale_column_row")
NORM_ONLY = ("rms_bf16", "eps_dropped", "eps_1e-5", "rms_half_dims", "qk_norm_weights_swapped",
             "weight_halves_swapped", "policies_swapped")


def gamma(d):
    return d * U / (1 - d * U)


# ---- launch predicate of csrc/rope.cu launch() ---------------------------------------------------
def launch_path(geom, fp8, misaligned=()):
    """("d128", 1) or ("generic", kCH) for a call whose pointers are 16-byte aligned except the
    ones named in `misaligned` (each a pointer of the aligned16 test of launch())."""
    dqk, dv = geom["dqk"], geom["dv"]
    ob = 1 if fp8 else 2
    if (dqk == 128 and dv % 16 == 0 and not misaligned and (geom["k_stride"] * ob) % 16 == 0
            and (geom["v_stride"] * ob) % 16 == 0):
        return "d128", 1
    ch = (dqk // 2 + 63) // 64
    return "generic", 1 if ch <= 1 else (2 if ch <= 2 else 4)


def generic_v_vector_rows(geom, fp8, rows, qkv_byte_offset=0, out_v=False):
    """Per row: does the generic kernel take its 16-byte V path (else the scalar one)?"""
    hq, hkv, dqk, dv = geom["hq"], geom["hkv"], geom["dqk"], geom["dv"]
    n = hkv * dv
    row_elems = hq * dqk + hkv * (dqk + dv)
    src = qkv_byte_offset + 2 * (np.arange(rows) * row_elems + (hq + hkv) * dqk)
    ob = 1 if fp8 else 2
    # the destination: a slot (v_off + cb * stride + pb * n) or a row of out_v (row * n)
    dst_ok = (ob * n) % (8 if fp8 else 16) == 0 and (out_v or (
        (ob * geom["v_stride"]) % 16 == 0 and (ob * geom["v_off"]) % 16 == 0))
    return (n % 8 == 0) & (src % 16 == 0) & dst_ok


def sum_terms(path, kch):
    return 4 * kch + 5


# ---- rows ----------------------------------------------------------------------------------------
def positions(seqlen, q_index, rows):
    """(pos, req) per row as the kernel finds them; pos = -1 for a row no request owns."""
    seqlen, q_index = np.asarray(seqlen, np.int64), np.asarray(q_index, np.int64)
    nreq = seqlen.shape[0]
    row = np.arange(rows)
    req = np.searchsorted(q_index, row, side="right") - 1
    ok = (req >= 0) & (req < nreq)
    rq = np.clip(req, 0, nreq - 1)
    q0, q1 = q_index[rq], q_index[rq + 1]
    ok &= (row >= q0) & (row < q1)
    pos = seqlen[rq] - (q1 - q0) + (row - q0)
    ok &= pos >= 0
    return np.where(ok, pos, -1), np.where(ok, rq, -1)


def _f64(t):
    import torch

    if isinstance(t, torch.Tensor):
        t = t.detach().cpu()
        return t.to(torch.float64).numpy()
    return np.asarray(t, np.float64)


def bits(t):
    """Raw bits of a bf16 (uint16) or 1-byte (uint8) tensor or array."""
    import torch

    if isinstance(t, torch.Tensor):
        t = t.detach().cpu().contiguous()
        return t.view(torch.int16).numpy().view(np.uint16) if t.element_size() == 2 else \
            t.view(torch.uint8).numpy()
    return np.asarray(t)


def split_heads(qkv, geom):
    """fp64 q [rows, Hq, D], k [rows, Hkv, D], bf16 bits of v [rows, Hkv * Dv]."""
    hq, hkv, dqk = geom["hq"], geom["hkv"], geom["dqk"]
    x = _f64(qkv)
    rows = x.shape[0]
    q = x[:, :hq * dqk].reshape(rows, hq, dqk)
    k = x[:, hq * dqk:(hq + hkv) * dqk].reshape(rows, hkv, dqk)
    v = bits(qkv)[:, (hq + hkv) * dqk:]
    return q, k, v


# ---- fp64 reference and bound --------------------------------------------------------------------
def _rotate(x, c, s):
    h = x.shape[-1] // 2
    a, b = x[..., :h], x[..., h:]
    y = np.concatenate([a * c - b * s, b * c + a * s], -1)
    t = np.concatenate([np.abs(a * c) + np.abs(b * s), np.abs(b * c) + np.abs(a * s)], -1)
    return y, t


def _e_a(e_s):
    e_m = (1 + e_s) * (1 + U) ** 2 - 1
    e_r = (1 + RSQRT_REL) * (1 - e_m) ** -0.5 - 1
    return (1 + e_r) * (1 + U) ** 2 - 1


def reference(x, cs, w, policy, d_terms):
    """fp64 y and bound b for heads x [rows, H, D] (fp64 of bf16) at table rows cs [rows, D]."""
    D = x.shape[-1]
    h = D // 2
    c, s = cs[:, None, :h], cs[:, None, h:]
    g2, gd = gamma(2), gamma(d_terms)
    if policy == 0:
        y, t = _rotate(x, c, s)
        return y, g2 * t + TINY
    w = np.asarray(w, np.float64)
    if policy == 2:
        r = 1 / np.sqrt((x * x).sum(-1, keepdims=True) / D + EPS)
        y, T = _rotate(x * r * w, c, s)
        return y, ((1 + _e_a(gd)) * (1 + g2) - 1) * T + TINY
    y0, t = _rotate(x, c, s)
    S = (y0 * y0).sum(-1, keepdims=True)
    delta = g2 * (t * (2 * np.abs(y0) + g2 * t)).sum(-1, keepdims=True)
    e_a = _e_a(delta / np.maximum(S, 1e-300) * (1 + gd) + gd)
    R = w / np.sqrt(S / D + EPS)
    return y0 * R, np.abs(R) * (g2 * t * (1 + e_a) + e_a * np.abs(y0)) + TINY


def bf16_rn(v):
    """float64 -> nearest bf16 value (ties to even), as float64 (normal range)."""
    b = np.ascontiguousarray(v, np.float64).view(np.uint64)
    lsb = (b >> np.uint64(45)) & np.uint64(1)
    b = (b + np.uint64((1 << 44) - 1) + lsb) & ~np.uint64((1 << 45) - 1)
    return b.view(np.float64)


def bf16_value(b16):
    return (np.asarray(b16, np.uint16).astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def check_bf16(b16, y, b):
    """(unexplained, explained flips) of kernel bf16 bits against y with fp32 bound b."""
    k = bf16_value(b16)
    ok = (k >= bf16_rn(y - b)) & (k <= bf16_rn(y + b))
    return int((~ok).sum()), int((ok & (k != bf16_rn(y))).sum())


def _fp8_bound(y, b, mult):
    v = y * mult
    return v, abs(mult) * (b * (1 + U) + U * np.abs(y)) + TINY


def _f32(x):
    return float(np.float32(x))


def rcp32(x):
    """__frcp_rn: the fp32 reciprocal, correctly rounded."""
    return float(np.float32(1) / np.float32(x))


# ---- the check of one call -----------------------------------------------------------------------
def grade(inp, out, fp8, path, fp8_args=None, before=None):
    """Check one call. inp: make_exact_inputs' dict (qkv may be any bf16 tensor of the same
    values); out: dict of what the call produced -- "q" (bits [rows, Hq, D]), "cache" (flat
    buffer bits after the call) or "out_k" / "out_v" (bits [rows, Hkv, D] / [rows, Hkv * Dv]),
    "q_scale" (fp32, fp8 quant_policy 1); before: the flat cache bits before the call.
    fp8_args: dict(k_scale, v_scale, quant_policy, upper_max, q_scale_inv).
    Returns {component: unexplained count, "flips_<component>": explained flips}."""
    geom = inp["geom"]
    hq, hkv, D, dv, page = geom["hq"], geom["hkv"], geom["dqk"], geom["dv"], geom["page"]
    rows = inp["qkv"].shape[0]
    pos, req = positions(inp["num_seqlen"], inp["q_index"], rows)
    live = np.nonzero(pos >= 0)[0]
    p, rq = pos[live], req[live]
    xq, xk, v16 = split_heads(inp["qkv"], geom)
    cs = _f64(inp["cos_sin"])[p]
    d = sum_terms(*path)
    pol = inp["policy"]
    yq, bq = reference(xq[live], cs, _f64(inp["q_norm_w"]) if pol else None, pol, d)
    yk, bk = reference(xk[live], cs, _f64(inp["k_norm_w"]) if pol else None, pol, d)
    res = {}

    def put(name, r):
        res[name], res["flips_" + name] = r

    # ---- Q ----
    q = np.asarray(out["q"])[live]
    if not fp8:
        put("q", check_bf16(q, yq, bq))
    elif fp8_args["quant_policy"] == 2:
        mult = _f32(fp8_args["q_scale_inv"])
        put("q", check_codes_within(q, *_fp8_bound(yq, bq, mult)))
    else:
        um = _f32(fp8_args["upper_max"])
        qs_all = np.asarray(out["q_scale"], np.float64)
        if inp["is_prefill"]:
            q0 = np.asarray(inp["q_index"], np.int64)[rq]
            qs = qs_all[rq[:, None], np.arange(hq)[None, :], (live - q0)[:, None]]
        else:
            qs = qs_all[live]
        lo = np.max(np.maximum(np.abs(yq) - bq, 0), -1) / um * (1 - U) - TINY
        hi = np.max(np.abs(yq) + bq, -1) / um * (1 + U) + TINY
        res["q_scale"] = int((~((qs >= lo) & (qs <= hi))).sum())
        mult = np.where(qs > 0, np.float32(1) / np.where(qs > 0, qs, 1).astype(np.float32), 0)
        mult = mult.astype(np.float64)[..., None]
        v, b = yq * mult, np.abs(mult) * (bq * (1 + U) + U * np.abs(yq)) + TINY
        put("q", check_codes_within(q, v, b))

    # ---- K and V of every live row, then where they went ----
    v_bits = v16[live]
    if fp8:
        mk = rcp32(fp8_args["k_scale"])
        vv = (v_bits.astype(np.uint32) << 16).view(np.float32) * np.float32(rcp32(fp8_args["v_scale"]))
        v_want = e4m3_code(vv.astype(np.float64))
    else:
        mk = 1.0
        v_want = v_bits

    def check_k(kb):
        if fp8:
            return check_codes_within(kb, *_fp8_bound(yk, bk, mk))
        return check_bf16(kb, yk, bk)

    if "out_k" in out:
        put("k", check_k(np.asarray(out["out_k"])[live]))
        res["v"] = int((np.asarray(out["out_v"])[live] != v_want).sum())
        res["cache"] = int((np.asarray(out["cache"]) != before).sum())
        return res

    cache = np.asarray(out["cache"])
    kv_idx = np.asarray(inp["kv_indices"], np.int64)
    cb = kv_idx[rq, p // page]
    pb = p % page
    ks = geom["k_off"] + cb * geom["k_stride"] + pb * hkv * D
    vs = geom["v_off"] + cb * geom["v_stride"] + pb * hkv * dv
    kidx = ks[:, None] + np.arange(hkv * D)[None, :]
    vidx = vs[:, None] + np.arange(hkv * dv)[None, :]
    put("k", check_k(cache[kidx].reshape(len(live), hkv, D)))
    res["v"] = int((cache[vidx] != v_want).sum())
    owned = np.zeros(cache.shape[0], bool)
    owned[kidx.ravel()] = True
    owned[vidx.ravel()] = True
    # tails: the slots after each request's last token, in that token's page
    tail = np.zeros(cache.shape[0], bool)
    last = np.nonzero(p == np.asarray(inp["num_seqlen"], np.int64)[rq] - 1)[0]
    for i in last:
        n0, n1 = (pb[i] + 1), page
        tail[geom["k_off"] + cb[i] * geom["k_stride"] + n0 * hkv * D:
             geom["k_off"] + cb[i] * geom["k_stride"] + n1 * hkv * D] = True
        tail[geom["v_off"] + cb[i] * geom["v_stride"] + n0 * hkv * dv:
             geom["v_off"] + cb[i] * geom["v_stride"] + n1 * hkv * dv] = True
    res["tail"] = int((cache[tail & ~owned] != 0).sum())
    rest = ~(owned | tail)
    res["untouched"] = int((cache[rest] != before[rest]).sum())
    return res


def failed(res):
    return {k: v for k, v in res.items() if not k.startswith("flips") and v}


# ---- fp32 emulation of the kernels, with named bugs ----------------------------------------------
def _bf16_bits(x32):
    b = np.ascontiguousarray(x32, np.float32).view(np.uint32)
    return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)


def _lane_ssq(x, path, kch):
    """fp32 sum of squares of x [..., D] in the kernel's order: per-lane sums, xor butterfly."""
    D = x.shape[-1]
    h = D // 2
    if path == "d128":
        sq = x.reshape(*x.shape[:-1], 32, 4)  # lane l owns dims 4l .. 4l+3
        s = ((sq[..., 0] * sq[..., 0] + sq[..., 1] * sq[..., 1]) + sq[..., 2] * sq[..., 2]) \
            + sq[..., 3] * sq[..., 3]
    else:
        pad = np.zeros((*x.shape[:-1], kch * 64 - h), np.float32)
        lo = np.concatenate([x[..., :h], pad], -1).reshape(*x.shape[:-1], kch, 32, 2)
        hi = np.concatenate([x[..., h:], pad], -1).reshape(*x.shape[:-1], kch, 32, 2)
        s = np.zeros((*x.shape[:-1], 32), np.float32)
        for c in range(kch):
            a, b = lo[..., c, :, :], hi[..., c, :, :]
            s = s + (((a[..., 0] * a[..., 0] + a[..., 1] * a[..., 1]) + b[..., 0] * b[..., 0])
                     + b[..., 1] * b[..., 1])
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        s = s + s[..., lane ^ o]
    return s[..., :1]


def _emulate_heads(x, cs, w, policy, path, kch, mutation):
    """fp32 rotated (normalised) heads x [rows, H, D]."""
    D = x.shape[-1]
    h = D // 2
    c, s = cs[:, None, :h], cs[:, None, h:]
    if mutation == "cos_sin_swapped":
        c, s = s, c
    f = np.float32

    def rms(v):
        if mutation == "rms_half_dims":
            ss, dd = _lane_ssq(np.concatenate([v[..., :h], 0 * v[..., :h]], -1), path, kch), f(h)
        else:
            ss, dd = _lane_ssq(v, path, kch), f(D)
        eps = {"eps_dropped": f(0), "eps_1e-5": f(1e-5)}.get(mutation, f(EPS))
        r = (1 / np.sqrt((ss / dd + eps).astype(np.float64))).astype(f)
        if mutation == "rms_bf16":
            r = bf16_value(_bf16_bits(r)).astype(f)
        ww = np.roll(w, h) if mutation == "weight_halves_swapped" else w
        return v * (r * ww.astype(f))

    if policy == 2:
        x = rms(x)
    if mutation == "gptj_pairs":
        a, b = x[..., 0::2], x[..., 1::2]
        ci, si = cs[:, None, :h], cs[:, None, h:]
        y = np.empty_like(x)
        y[..., 0::2], y[..., 1::2] = a * ci - b * si, b * ci + a * si
    else:
        a, b = x[..., :h], x[..., h:]
        sg = -1 if mutation == "rotation_sign" else 1
        y = np.concatenate([a * c - sg * (b * s), b * c + sg * (a * s)], -1).astype(f)
    if policy == 1:
        y = rms(y)
    return y.astype(f)


def emulate(inp, fp8, path, mutation=None, fp8_args=None, bypass=False, before=None):
    """What a kernel of `path` (("d128", 1) / ("generic", kCH)) computes, in fp32 numpy, with an
    optional bug from MUTATIONS. Returns the `out` dict that grade() takes."""
    geom = inp["geom"]
    hq, hkv, D, dv, page = geom["hq"], geom["hkv"], geom["dqk"], geom["dv"], geom["page"]
    rows = inp["qkv"].shape[0]
    pos, req = positions(inp["num_seqlen"], inp["q_index"], rows)
    live = np.nonzero(pos >= 0)[0]
    p, rq = pos[live], req[live]
    table = np.asarray(inp["cos_sin"], np.float32)
    pt = p + {"pos+1": 1, "pos-1": -1}.get(mutation, 0)
    cs = table[np.clip(pt, 0, table.shape[0] - 1)]
    xq, xk, v16 = split_heads(inp["qkv"], geom)
    pol = inp["policy"]
    if mutation == "policies_swapped" and pol:
        pol = 3 - pol
    qw, kw = np.asarray(inp["q_norm_w"], np.float32), np.asarray(inp["k_norm_w"], np.float32)
    if mutation == "qk_norm_weights_swapped":
        qw, kw = kw, qw
    kind, kch = path
    yq = _emulate_heads(xq[live].astype(np.float32), cs, qw, pol, kind, kch, mutation)
    yk = _emulate_heads(xk[live].astype(np.float32), cs, kw, pol, kind, kch, mutation)
    f = np.float32
    out = {}
    q_bits = np.zeros((rows, hq, D), np.uint8 if fp8 else np.uint16)
    if fp8:
        if fp8_args["quant_policy"] == 1:
            um = FP8_MAX if mutation == "upper_max_ignored" else _f32(fp8_args["upper_max"])
            qs = (np.abs(yq).max(-1) / f(um)).astype(f)
            mult = np.where(qs > 0, f(1) / np.where(qs > 0, qs, 1), 0).astype(f)[..., None]
            if inp["is_prefill"]:
                pad = (inp["max_seqlens"] + 127) // 128 * 128
                buf = np.full((geom_nreq(inp), hq, pad), np.nan, f)
                q0 = np.asarray(inp["q_index"], np.int64)[rq]
                col = live if mutation == "q_scale_column_row" else live - q0
                okc = col < pad
                buf[rq[okc][:, None], np.arange(hq)[None, :], col[okc][:, None]] = qs[okc]
            else:
                buf = np.full((rows, hq), np.nan, f)
                buf[live] = qs
            out["q_scale"] = buf
        else:
            mult = f(fp8_args["q_scale_inv"])
        q_bits[live] = e4m3_code((yq * mult).astype(f).astype(np.float64))
        mk = f(fp8_args["k_scale"]) if mutation == "k_times_scale" else f(rcp32(fp8_args["k_scale"]))
        vsc = fp8_args["k_scale"] if mutation == "v_with_k_scale" else fp8_args["v_scale"]
        k_out = e4m3_code((yk * mk).astype(f).astype(np.float64))
        vv = (v16[live].astype(np.uint32) << 16).view(f) * f(rcp32(vsc))
        v_out = e4m3_code(vv.astype(np.float64))
    else:
        q_bits[live] = _bf16_bits(yq)
        k_out, v_out = _bf16_bits(yk), v16[live]
    out["q"] = q_bits
    cache = np.array(before, copy=True)
    out["cache"] = cache
    if bypass:
        sent = np.uint8(0x7F) if fp8 else np.uint16(0x7FC0)
        out["out_k"] = np.full((rows, hkv, D), sent)
        out["out_v"] = np.full((rows, hkv * dv), sent)
        out["out_k"][live], out["out_v"][live] = k_out, v_out
        return out
    kv_idx = np.asarray(inp["kv_indices"], np.int64)
    cb, pb = kv_idx[rq, p // page], p % page
    kst = page * hkv * D if mutation == "dense_page_stride" else geom["k_stride"]
    vst = page * hkv * dv if mutation == "dense_page_stride" else geom["v_stride"]
    k0 = geom["k_off"] + cb * kst
    v0 = geom["v_off"] + cb * vst
    cache[(k0 + pb * hkv * D)[:, None] + np.arange(hkv * D)] = k_out.reshape(len(live), -1)
    cache[(v0 + pb * hkv * dv)[:, None] + np.arange(hkv * dv)] = v_out.reshape(len(live), -1)
    seq = np.asarray(inp["num_seqlen"], np.int64)[rq]
    zero_rows = np.arange(len(live)) if mutation == "tail_every_page" else np.nonzero(p == seq - 1)[0]
    for i in zero_rows:
        first = pb[i] + (0 if mutation == "tail_from_pb" else 1)
        for s_ in range(first, page):
            kk = k0[i] + s_ * hkv * D
            cache[kk:kk + (D if mutation == "k_tail_head0" else hkv * D)] = 0
            cache[v0[i] + s_ * hkv * dv:v0[i] + (s_ + 1) * hkv * dv] = 0
    return out


def geom_nreq(inp):
    return int(np.asarray(inp["num_seqlen"]).shape[0])


def mutations_for(inp, fp8, fp8_args=None):
    """The MUTATIONS a cache-path call on `inp` can express (the others do not change its result)."""
    geom = inp["geom"]
    rows = inp["qkv"].shape[0]
    pos, req = positions(inp["num_seqlen"], inp["q_index"], rows)
    live = pos >= 0
    p, rq = pos[live], req[live]
    seq = np.asarray(inp["num_seqlen"], np.int64)[rq]
    q0 = np.asarray(inp["q_index"], np.int64)[rq]
    out = []
    for m in MUTATIONS:
        if m in FP8_ONLY and not fp8:
            continue
        if m in NORM_ONLY and inp["policy"] == 0:
            continue
        if m == "upper_max_ignored" and (fp8_args["quant_policy"] != 1 or fp8_args["upper_max"] == FP8_MAX):
            continue
        if m == "q_scale_column_row" and not (inp["is_prefill"] and fp8_args["quant_policy"] == 1
                                              and (q0 > 0).any()):
            continue
        if m == "k_tail_head0" and geom["hkv"] == 1:
            continue
        if m == "dense_page_stride" and geom["layout"] != "combined":
            continue
        if m == "tail_every_page" and not ((p < seq - 1) & ((p + 1) % geom["page"] != 0)).any():
            continue
        out.append(m)
    return out
