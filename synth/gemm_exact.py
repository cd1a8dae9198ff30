"""Inputs for oracle/gemm_exact.py: the route GEMM and the stand-alone grouped FP8 GEMMs, built so
that a kernel that is subtly wrong cannot pass the per-element check.

Route GEMM. x is bf16 randn. Three regimes for the low part:
  split  the real use: w fp32 randn, w_high = bf16(w), w_low = bf16((w - w_high) / scale),
         scale = 1/256 (the low term is below half a bf16 ulp of the output);
  indep  scale = 1 with an independent w_low of w_high's magnitude, so dropping or mis-scaling
         the low term moves a bf16 output by many ulps;
  neg    scale = -0.37 (negative, not a power of two) with an independent w_low.
Where n < k and n <= 512, a few rows are projected onto the null space of the effective weight
before their bf16 rounding, so |y| << S on those rows (strong cancellation); they are listed in
`cancel_rows`. Shapes cover TN = 64 and 128 tiles, m around every 128-row boundary and k with a
ragged last step, one step, and step counts that 2 / 4 / 8 do not divide: k = 72 and 200 leave whole
CTAs of a cluster of 4 or 8 with no step, k = 960 (15 steps) keeps every CTA busy with a short last.

Grouped GEMMs. Normal-range e4m3 data (sign * 2^U(-4, 4)) with scales that make outputs O(1);
every group has its own y_scale (per-tensor) or its own weight-scale blocks (blockwise), so a
neighbouring group's scale shows. The every-code cases put one e4m3 code per X row (or per W row) at
a K position that walks over the block, all 254 finite codes including subnormals and +-448, against
power-of-two partners and power-of-two y_scale: every output is one exact product.
"""
import functools

import torch

from oracle import moe_exact as ox
from oracle.gemm_exact import reformat_layout
from synth.moe import _E4M3_MS, _normal_e4m3, _signed_scale

ROUTE_CASES = [
    dict(m=1, n=64, k=8, regime="split"),
    dict(m=7, n=192, k=56, regime="indep"),
    dict(m=127, n=320, k=64, regime="neg"),
    dict(m=128, n=128, k=72, regime="split"),
    dict(m=129, n=256, k=200, regime="indep"),
    dict(m=255, n=2048, k=1000, regime="neg"),
    dict(m=1000, n=192, k=4096, regime="indep"),
    dict(m=12303, n=64, k=7168, regime="split"),
    dict(m=129, n=7168, k=200, regime="indep"),
    dict(m=255, n=320, k=7168, regime="neg"),
    dict(m=1000, n=128, k=1000, regime="split"),
    dict(m=7, n=2048, k=4096, regime="neg"),
    dict(m=1000, n=256, k=960, regime="neg"),
]


def route_tag(c):
    return f"m{c['m']}_n{c['n']}_k{c['k']}_{c['regime']}"


@functools.lru_cache(maxsize=16)
def _route_cached(m, n, k, regime, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((m, k), generator=g)
    if regime == "split":
        scale = 1.0 / 256
        w = torch.randn((n, k), generator=g)
        w_high = w.to(torch.bfloat16)
        w_low = ((w - w_high.float()) / scale).to(torch.bfloat16)
    else:
        scale = 1.0 if regime == "indep" else -0.37
        w_high = torch.randn((n, k), generator=g).to(torch.bfloat16)
        w_low = torch.randn((n, k), generator=g).to(torch.bfloat16)
    cancel = []
    if n < k and n <= 512:
        weff = w_high.double() + scale * w_low.double()
        cancel = sorted({0, m // 2, m - 1})
        z = x[cancel].double()
        coef = torch.linalg.solve(weff @ weff.t(), weff @ z.t())  # [n, r]
        x[cancel] = (z - (weff.t() @ coef).t()).float()
    return dict(x=x.to(torch.bfloat16), w_high=w_high, w_low=w_low, scale=scale,
                cancel_rows=torch.tensor(cancel, dtype=torch.long))


def make_route_inputs(c, seed=7):
    return _route_cached(c["m"], c["n"], c["k"], c["regime"], seed)


# ------------------------------------------------------------------------------------------------
# grouped
# ------------------------------------------------------------------------------------------------
def _layout(rows, gapped, stride=None):
    seqlens = torch.tensor(rows, dtype=torch.int32)
    G = len(rows)
    if gapped:  # DeepEP: group g owns rows g * stride .. g * stride + stride - 1
        stride = stride or max(max(rows), 1)
        cu = torch.arange(G + 1, dtype=torch.int32) * stride
    else:
        cu = torch.zeros(G + 1, dtype=torch.int32)
        cu[1:] = torch.cumsum(seqlens, 0)
    return seqlens, cu, int(cu[-1])


def _pow2(shape, g, lo=-3, hi=3):
    e = torch.randint(lo, hi + 1, shape, generator=g).float()
    s = torch.randint(0, 2, shape, generator=g).float() * 2 - 1
    return (s * torch.exp2(e)).to(torch.float8_e4m3fn)


def finite_codes():
    """The 254 finite e4m3 codes (every byte but the NaNs 0x7F and 0xFF), as e4m3."""
    b = torch.tensor([c for c in range(256) if c & 0x7F != 0x7F], dtype=torch.uint8)
    return b.view(torch.float8_e4m3fn)


def _code_rows(nrows, K, g):
    """[nrows, K] e4m3: row i holds finite code i (cycled) at K position (i * 37 + shift) % K."""
    codes = finite_codes()
    out = torch.zeros((nrows, K), dtype=torch.uint8)
    shift = int(torch.randint(0, K, (1,), generator=g))
    for i in range(nrows):
        out[i, (i * 37 + shift) % K] = codes.view(torch.uint8)[i % codes.numel()]
    return out.view(torch.float8_e4m3fn)


# per-tensor cases: (tag, rows per group, gapped, n, k, kind)
PERTENSOR_CASES = [
    ("codes_x", [127, 0, 127], False, 64, 144, "codes_x"),
    ("codes_w", [65, 63], False, 256, 128, "codes_w"),
    ("g8_edges", [0, 1, 63, 64, 65, 127, 128, 129], False, 192, 48, "normal"),
    ("g8_gapped", [300, 0, 129, 1, 64, 0, 65, 127], True, 320, 1008, "normal"),
    ("g128_gapped", "g128", True, 64, 192, "normal"),
    ("g512", "g512", False, 64, 16, "normal"),
    ("all_empty", [0, 0, 0, 0], False, 64, 16, "normal"),
    ("g1_big", [129], False, 4096, 7168, "normal"),
]

SCATTER_CASES = [
    ("scatter_edges", [1, 64, 65, 0], 192, 144),
    ("scatter_g8", [0, 1, 63, 64, 65, 127, 128, 129], 64, 48),
]

# blockwise: the standalone layouts, and one DeepEP round trip per granule bucket of the GEMM's rule
BLOCKWISE_CASES = [
    ("bw_g8_edges", [0, 1, 63, 64, 65, 127, 128, 129], False, 384, 384, None),
    ("bw_g512", "g512", False, 128, 128, None),
    ("bw_g1_k512", [200], False, 256, 512, None),
]
ROUNDTRIP_AVGS = [5, 12, 30, 40, 60, 80, 110, 140, 200]


def _rows_spec(spec, g):
    if spec == "g128":
        return torch.randint(0, 6, (128,), generator=g).tolist()
    if spec == "g512":
        return torch.randint(0, 4, (512,), generator=g).tolist()
    return list(spec)


def _distinct(G):
    """Distinct per-group factors in [0.6, 1.4]; neighbours differ by >= 0.3."""
    return torch.tensor([0.6 + 0.8 * ((g * 0.6180339887) % 1.0) for g in range(G)])


def make_pertensor_case(case, seed=11):
    tag, spec, gapped, n, k, kind = case
    g = torch.Generator().manual_seed(seed)
    rows = _rows_spec(spec, g)
    seqlens, cu, M = _layout(rows, gapped)
    G = len(rows)
    M = max(M, 8)  # an all-empty problem still has rows, which must stay unwritten
    if kind == "codes_x":
        x = _code_rows(M, k, g)
        w = _pow2((G, n, k), g)
        ys = torch.exp2(torch.tensor([-1.0, 1.0, 2.0]))[:G]
    elif kind == "codes_w":
        x = _pow2((M, k), g)
        w = torch.stack([_code_rows(n, k, g) for _ in range(G)])
        ys = torch.exp2(torch.tensor([1.0, -2.0]))[:G]
    else:
        x = _normal_e4m3((M, k), g)
        w = torch.stack([_normal_e4m3((n, k), g) for _ in range(G)])
        ys = _distinct(G) / (_E4M3_MS * k ** 0.5)
    return dict(tag=tag, x=x, w=w, seqlens=seqlens, cu_seqlens=cu, y_scale=ys.float(), gapped=gapped)


def make_scatter_case(case, seed=12):
    tag, rows, n, k = case
    g = torch.Generator().manual_seed(seed)
    seqlens, cu, M = _layout(rows, False)
    G = len(rows)
    pool_rows = M + 37
    pool = _normal_e4m3((pool_rows, k), g)
    idx = torch.arange(M - 1, -1, -1)  # reversed
    idx[1::5] = idx[0::5][:idx[1::5].numel()]  # repeated
    idx[0] = pool_rows - 1  # the pool's last row
    specials = [-1, pool_rows, pool_rows + 5, -7]  # clamped to the first / last pool row
    idx[2:2 + len(specials)] = torch.tensor(specials)[:max(0, M - 2)]
    w = torch.stack([_normal_e4m3((n, k), g) for _ in range(G)])
    ys = _distinct(G) / (_E4M3_MS * k ** 0.5)
    return dict(tag=tag, pool=pool, row_indices=idx.to(torch.int32), w=w, seqlens=seqlens,
                cu_seqlens=cu, y_scale=ys.float())


def _blockwise_common(rows, gapped, n, k, g, stride=None, kpad_extra=0):
    seqlens, cu, M = _layout(rows, gapped, stride)
    G = len(rows)
    KB = k // 128
    kpad4 = (KB + 3) // 4 * 4 + kpad_extra
    x = _normal_e4m3((M, k), g)
    w = torch.stack([_normal_e4m3((n, k), g) for _ in range(G)])
    x_scale = _signed_scale((M, KB), g).float()
    ws = _signed_scale((G, n // 128, kpad4), g) / (_E4M3_MS * (k * 1.08) ** 0.5)
    ws[:, :, KB:] = float("nan")  # padding entries: a kernel that reads one shows NaN
    return dict(x=x, w=w, seqlens=seqlens, cu_seqlens=cu, x_scale=x_scale, w_scale=ws.float(),
                kpad4=kpad4)


def make_blockwise_case(case, seed=13):
    """Standalone blockwise case: the transposed activation scales are laid out with the GEMM's
    granule (NaN in every unused column)."""
    tag, spec, gapped, n, k, avg = case
    g = torch.Generator().manual_seed(seed)
    rows = _rows_spec(spec, g)
    d = _blockwise_common(rows, gapped, n, k, g, kpad_extra=4 if k == 512 else 0)
    avg = avg if avg is not None else max(1, sum(rows) // len(rows))
    gran = ox.scale_granule(avg)
    lay = reformat_layout(d["x_scale"], d["seqlens"], d["cu_seqlens"], gran)
    m_pad = (int(lay.size(1)) + gran + 3) // 4 * 4
    xs_t = torch.full((lay.size(0), m_pad), float("nan"))
    xs_t[:, :lay.size(1)] = lay
    return dict(d, tag=tag, avg=avg, granule=gran, xscale_t=xs_t)


def make_roundtrip_case(avg, seed=14):
    """DeepEP layout for a given avg: 4 groups at a fixed row stride (a multiple of every granule),
    one of them empty, the others around avg rows and not multiples of the granule (the first
    one such that the old reformat granule, 64 for avg > 48, pads it differently)."""
    g = torch.Generator().manual_seed(seed + avg)
    rows = [max(1, avg - avg // 5), avg + 3, 0, avg + 2]
    stride = 256 if avg > 144 else 192
    d = _blockwise_common(rows, True, 256, 256, g, stride=stride)
    return dict(d, tag=f"roundtrip_avg{avg}", avg=avg, granule=ox.scale_granule(avg))
