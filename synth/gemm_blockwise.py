"""Inputs for oracle/gemm_blockwise.py: the dense blockwise FP8 GEMM and the 1x128 quantiser, built so
that a kernel that is subtly wrong cannot pass the per-element check.

GEMM operands. x and w are e4m3 codes drawn uniformly from all 254 finite codes (every code appears
in both operands, subnormals and +-448 included), except row 0 of x, which holds subnormal codes
only: its outputs come from subnormal products alone, so decoding them as normals shows. Scales
are signed and log-uniform over 2^[-6, 6], drawn per (row, K block) and per (N block, K block), so
a scale read from the wrong row, K block or N block moves an output by far more than its bound.
Where N < K, the last rows of x are the e4m3 quantisation of vectors projected onto the null space
of the dequantised weight (|y| << S: the rows where accumulation error is not hidden by the output's
magnitude); they are listed in `cancel_rows`.

CASES cover ragged N (576, 1000, 2112), M that is not a multiple of the tile, a single K block,
K-block counts that 2, 4 and 8 do not divide, more tiles than SMs (the persistent loop), and each
K split the launcher picks on an H100 (`split`, the value the CPU emulation uses; the GPU test
takes hpc_gemm_blockwise_fp8_config's).

Quantiser inputs. bf16 randn rows whose 128-column blocks have magnitudes 2^U(-20, 20), with
all-zero blocks, blocks of amax ~1e-6 (where the +1e-8 of 1 / (sc + 1e-8) matters) and blocks near
the top of the bf16 range.
"""
import functools

import torch

from oracle import gemm_blockwise as ob

CASES = [
    dict(m=200, n=1000, k=128, split=1),    # one K block, ragged N, ragged M
    dict(m=1100, n=2112, k=256, split=1),   # 153 tiles: the persistent loop
    dict(m=1, n=2112, k=640, split=2),      # 5 K blocks over 2
    dict(m=70, n=2112, k=1152, split=4),    # 9 K blocks over 4
    dict(m=3, n=576, k=2176, split=8),      # 17 K blocks over 8, null-space rows
    dict(m=130, n=256, k=1024, split=4),    # two m-tiles, null-space rows
]


def tag(c):
    return f"m{c['m']}_n{c['n']}_k{c['k']}"


_FINITE = torch.tensor([b for b in range(256) if (b & 0x7F) != 0x7F], dtype=torch.uint8)
_SUBNORMAL = torch.tensor([s | b for s in (0, 0x80) for b in range(1, 8)], dtype=torch.uint8)


def _codes(rows, cols, g):
    """e4m3 [rows, cols]: uniform over the 254 finite codes, each of which appears when the tensor
    has at least 254 elements."""
    idx = torch.randint(0, _FINITE.numel(), (rows * cols,), generator=g)
    idx[:min(rows * cols, _FINITE.numel())] = torch.arange(min(rows * cols, _FINITE.numel()))
    idx = idx[torch.randperm(rows * cols, generator=g)]
    return _FINITE[idx].view(rows, cols).view(torch.float8_e4m3fn)


def _scales(shape, g):
    mag = torch.exp2(torch.empty(shape).uniform_(-6, 6, generator=g))
    sign = torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0)
    return (sign * mag).float()


def dequant_weight(w, ws):
    n = w.size(0)
    return w.float() * ws.repeat_interleave(128, 0)[:n].repeat_interleave(128, 1)


@functools.lru_cache(maxsize=8)
def _cached(m, n, k, seed):
    g = torch.Generator().manual_seed(seed)
    kb, nb = k // 128, (n + 127) // 128
    x = _codes(m, k, g)
    w = _codes(n, k, g)
    xs = _scales((m, kb), g)
    ws = _scales((nb, kb), g)
    sub = _SUBNORMAL[torch.randint(0, _SUBNORMAL.numel(), (k,), generator=g)]
    x.view(torch.uint8)[0] = sub
    cancel = torch.zeros(0, dtype=torch.long)
    if n < k and m >= 2:
        nc = min(2, m - 1)
        wd = dequant_weight(w, ws).double()
        v = torch.randn((nc, k), generator=g, dtype=torch.float64)
        q, _ = torch.linalg.qr(wd.t())  # orthonormal basis of the row space of w
        v = v - (v @ q) @ q.t()
        v = v / v.abs().max() * 300.0
        qx, qs = ob.quant(v.to(torch.bfloat16))
        cancel = torch.arange(m - nc, m)
        x[cancel] = qx
        xs[cancel] = qs
    return dict(x=x, xs=xs.contiguous(), w=w, ws=ws.contiguous(), cancel_rows=cancel)


def make_inputs(c, seed=0):
    """dict(x, xs, w, ws, cancel_rows) on the CPU."""
    return _cached(c["m"], c["n"], c["k"], seed)


def real_inputs(m, n, k, seed=0):
    """Operands of a projection shape: x from blockwise_quant of bf16 randn activations, w codes
    of a randn weight quantised per 128 x 128 block (amax / 448), ws its scales; (x, xs, w, ws)."""
    g = torch.Generator().manual_seed(seed)
    a = torch.randn((m, k), generator=g).to(torch.bfloat16)
    x, xs = ob.quant(a)
    nb, kb = (n + 127) // 128, k // 128
    wf = torch.randn((nb * 128, k), generator=g) * 0.02
    blk = wf.view(nb, 128, kb, 128)
    ws = (blk.abs().amax((1, 3)) / 448.0).float()
    w = (blk / ws[:, None, :, None]).clamp(-448, 448).view(nb * 128, k)[:n].to(torch.float8_e4m3fn)
    return x, xs, w.contiguous(), ws.contiguous()


def quant_input(m, k, seed=0, ld=None):
    """bf16 [m, k] (a view with row stride `ld` when given) with the special blocks listed above."""
    g = torch.Generator().manual_seed(seed)
    ld = k if ld is None else ld
    kb = k // 128
    base = torch.randn((m, ld), generator=g)
    mag = torch.exp2(torch.empty((m, kb)).uniform_(-20, 20, generator=g))
    base[:, :k] *= mag.repeat_interleave(128, 1)
    kind = torch.randint(0, 8, (m, kb), generator=g)
    blocks = base[:, :k].view(m, kb, 128)
    blocks[kind == 0] = 0.0
    blocks[kind == 1] = blocks[kind == 1] / blocks[kind == 1].abs().amax(-1, keepdim=True) * 1e-6
    blocks[kind == 2] = blocks[kind == 2].sign() * 3.0e38
    full = base.to(torch.bfloat16)
    return full[:, :k]
