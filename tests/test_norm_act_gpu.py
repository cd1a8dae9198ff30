"""GPU tests of hpc.fused_rmsnorm_with_scale and the masked per-expert activation quantisers
(reference tests/test_normalization.py, tests/test_act.py:62-174): the reference's fixtures and
shapes, a grid checked against the fp64 oracle's bound (oracle/normalization.py) and the kernel-way
masked oracle (oracle/masked_act.py), untouched invalid rows, and CUDA-graph replay."""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import masked_act as oact
from oracle import normalization as on
from synth import act as sa
from synth import normalization as sn

pytestmark = pytest.mark.gpu
G = Path(__file__).resolve().parent / "golden"


def _bf16(a):
    return torch.from_numpy(a).view(torch.bfloat16)


def _close(gt, my, atol, rtol):
    return torch.allclose(gt.float().cpu(), my.float().cpu(), atol=atol, rtol=rtol)


def _rows(T, H):
    """The rows the fp64 oracle checks: all of them up to 8 M elements, else a fixed spread."""
    if T * H <= (8 << 20):
        return torch.arange(T)
    return torch.unique(torch.cat([torch.arange(64), torch.arange(T - 64, T), torch.arange(0, T, 37)]))


def _run_norm(hpc, x, w, scale, eps):
    q = hpc.normalization.fused_rmsnorm_with_scale(x, w, scale=scale, eps=eps, is_moe=False)
    y32, q0, q1 = hpc.normalization.fused_rmsnorm_with_scale(x, w, scale=scale, eps=eps, is_moe=True)
    return q, (y32, q0, q1)


def _check_norm(hpc, x, w, scale, eps):
    q, moe = _run_norm(hpc, x, w, scale, eps)
    assert q.dtype == torch.float8_e4m3fn and q.shape == x.shape
    assert moe[0].dtype == torch.float32 and moe[2].shape == x.shape
    # is_moe only adds outputs: q0 is the same byte either way
    assert torch.equal(q.view(torch.uint8), moe[1].view(torch.uint8))
    rows = _rows(*x.shape).to(x.device)
    res = on.check(tuple(t[rows] for t in moe), x[rows], w, eps, scale, True)
    assert not on.failed(res), res
    return res


# ---- the reference's fixtures, at its tolerances and then tightly ---------------------------------
@pytest.mark.parametrize("H", [320, 4096, 5120])
@pytest.mark.parametrize("is_moe", [False, True])
def test_norm_golden(hpc, H, is_moe):
    z = np.load(G / f"norm_h{H}_{'moe' if is_moe else 'plain'}.npz")
    x, w = _bf16(z["x"]).cuda(), _bf16(z["w"]).cuda()
    sc, eps = torch.from_numpy(z["scale"]).cuda(), float(z["eps"][0])
    out = hpc.normalization.fused_rmsnorm_with_scale(x, w, scale=sc, eps=eps, is_moe=is_moe)
    y32, q0, q1 = out if is_moe else (torch.from_numpy(z["gt_fp32"]), out, out)
    assert _close(torch.from_numpy(z["gt_fp32"]), y32, 1e-8, 1e-5)
    assert _close(_bf16(z["gt"]), q0.to(torch.bfloat16), 0.15, 0.0125)
    assert _close(_bf16(z["gt2"]), q1.to(torch.bfloat16), 0.15, 0.0125)
    if not is_moe:
        sc = torch.cat([sc, sc])
    _check_norm(hpc, x, w, sc, eps)


@pytest.mark.parametrize("tag", ["a", "b"])
def test_masked_golden(hpc, tag):
    z = np.load(G / f"masked_act_{tag}.npz")
    gu, sc = _bf16(z["gate_up"]).cuda(), torch.from_numpy(z["scale"]).cuda()
    cnt, T = torch.from_numpy(z["num_per_expert"]).cuda(), int(z["T_max"][0])
    keep = sa.valid_rows(cnt.cpu(), T)
    my = hpc.masked_act_mul_and_quant(gu, sc, cnt).cpu()
    gt = torch.from_numpy(z["gt"]).view(torch.float8_e4m3fn)
    assert _close(gt.float()[keep], my.float()[keep], 0.15, 0.0125)
    bad, step = oact.fp8_mismatch(my[keep], gt[keep])
    assert bad <= 2 and step <= 1
    mb, ms = hpc.masked_act_mul_and_blockwise_quant(gu, cnt)
    gtb = torch.from_numpy(z["gt_block"]).view(torch.float8_e4m3fn)
    gts = torch.from_numpy(z["gt_scale"])
    assert _close(gtb.float()[keep], mb.float().cpu()[keep], 32, 0.0125)
    assert _close(gts[keep], ms.cpu()[keep], 0.15, 0.0125)
    # tightly: a few ulp from CUDA expf (oracle/masked_act.py SCALE_REL)
    assert ((ms.cpu()[keep] - gts[keep]).abs() <= oact.SCALE_REL * gts[keep].abs()).all()
    bad, step = oact.fp8_mismatch(mb.cpu()[keep], gtb[keep])
    assert bad <= max(2, 0.001 * gtb[keep].numel()) and step <= 1


# ---- RMSNorm grid -----------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [8, 264, 320, 1032, 2048, 4096, 5120, 7168, 8192, 16384])
@pytest.mark.parametrize("T", [1, 3, 17, 64, 1000, 8192])
def test_norm_grid(hpc, H, T):
    d = sn.make_inputs(T, H, seed=1, device="cuda")
    _check_norm(hpc, d["x"], d["w"], d["scale"], d["eps"])


@pytest.mark.parametrize("batch", [1, 2, 4, 5, 8, 14, 16, 17, 32, 64])
@pytest.mark.parametrize("H", [5120, 320, 4096])
def test_norm_reference_shapes(hpc, batch, H):
    # reference tests/test_normalization.py:31-66, both is_moe in one call of _check_norm
    torch.manual_seed(0)
    w = torch.rand((1, H), dtype=torch.bfloat16).cuda()
    x = torch.randn(batch, H, dtype=torch.bfloat16).cuda()
    sc = torch.tensor([2.5, 5.0], dtype=torch.float32).cuda()
    _check_norm(hpc, x, w, sc, 1e-6)
    y = on.rmsnorm(x, w, 1e-6)
    q, (y32, q0, q1) = _run_norm(hpc, x, w, sc, 1e-6)
    assert _close(torch.from_numpy(y).float(), y32, 1e-8, 1e-5)


def test_norm_default_scale_and_3d(hpc):
    d = sn.make_inputs(12, 256, seed=3, device="cuda")
    x = d["x"].reshape(3, 4, 256)
    q = hpc.fused_rmsnorm_with_scale(x, d["w"])  # CPU default scale [1.0], copied to the device
    assert q.shape == (3, 4, 256)
    res = on.check(q.reshape(12, 256), d["x"], d["w"], torch.finfo(torch.float32).eps,
                   torch.ones(1), False)
    assert not on.failed(res), res


# ---- masked activation quantisers ------------------------------------------------------------------
def _masked_call(hpc, d, blockwise):
    gu, cnt = d["gate_up"], d["num_per_expert"]
    N, C = gu.shape[0], gu.shape[1] // 2
    sent = sa.sentinel_outputs(N, C, device="cuda")
    out, osc = sent[0].clone(), sent[1].clone()
    if blockwise:
        r = hpc.masked_act_mul_and_blockwise_quant(gu, cnt, output=out, output_scale=osc)
        assert r[0].data_ptr() == out.data_ptr() and r[1].data_ptr() == osc.data_ptr()
    else:
        r = hpc.masked_act_mul_and_quant(gu, d["scale"], cnt, output=out)
        assert r.data_ptr() == out.data_ptr()
        osc = None
    return oact.masked_check(out, osc, gu, cnt, d["T_max"], sent, scale=d["scale"])


@pytest.mark.parametrize("E", [1, 8, 32])
@pytest.mark.parametrize("T_max", [1, 7, 336, 1024])
@pytest.mark.parametrize("blockwise", [False, True])
def test_masked_grid(hpc, E, T_max, blockwise):
    d = sa.make_inputs(E, T_max, 256, seed=2, device="cuda")
    res = _masked_call(hpc, d, blockwise)
    assert oact.masked_ok(res), res


@pytest.mark.parametrize("blockwise", [False, True])
def test_masked_reference_shape(hpc, blockwise):
    # reference tests/test_act.py:62-174: E 32, T_max 336, C 2048
    d = sa.make_inputs(32, 336, 2048, seed=4, device="cuda")
    res = _masked_call(hpc, d, blockwise)
    assert oact.masked_ok(res), res


def test_masked_full_equals_act_mul_and_quant(hpc):
    E, T, C = 8, 100, 1024
    d = sa.make_inputs(E, T, C, seed=5, device="cuda")
    cnt = torch.full((E,), T, dtype=torch.int32, device="cuda")
    a = hpc.masked_act_mul_and_quant(d["gate_up"], d["scale"], cnt)
    b = hpc.act_mul_and_quant(d["gate_up"], d["scale"], use_bf16_mul=False)
    assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def test_masked_default_outputs(hpc):
    d = sa.make_inputs(4, 16, 256, seed=6, device="cuda")
    q, s = hpc.masked_act_mul_and_blockwise_quant(d["gate_up"], d["num_per_expert"])
    assert q.shape == (64, 256) and s.shape == (64, 2) and s.dtype == torch.float32
    q = hpc.masked_act_mul_and_quant(d["gate_up"], d["scale"], d["num_per_expert"])
    assert q.shape == (64, 256) and q.dtype == torch.float8_e4m3fn


# ---- CUDA graphs -------------------------------------------------------------------------------------
def _graph(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn()
    return g, out


def test_graph_replay_norm(hpc):
    d = sn.make_inputs(64, 4096, seed=7, device="cuda")
    x, w, sc = d["x"].clone(), d["w"].clone(), d["scale"].clone()
    g, out = _graph(lambda: hpc.fused_rmsnorm_with_scale(x, w, 1e-6, sc, True))
    g2, out2 = _graph(lambda: hpc.fused_rmsnorm_with_scale(x, w, 1e-6, sc, False))
    n = sn.make_inputs(64, 4096, seed=8, device="cuda")
    x.copy_(n["x"])
    w.copy_(n["w"])
    sc.copy_(torch.tensor([0.02, 0.5], device="cuda"))
    g.replay()
    g2.replay()
    ref = hpc.fused_rmsnorm_with_scale(x, w, 1e-6, sc, True)
    torch.cuda.synchronize()
    for a, b in zip(out, ref):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))
    assert torch.equal(out2.view(torch.uint8), ref[1].view(torch.uint8))


@pytest.mark.parametrize("blockwise", [False, True])
def test_graph_replay_masked(hpc, blockwise):
    E, T, C = 8, 64, 512
    d = sa.make_inputs(E, T, C, seed=9, device="cuda")
    gu, cnt, sc = d["gate_up"].clone(), d["num_per_expert"].clone(), d["scale"].clone()
    if blockwise:
        g, out = _graph(lambda: hpc.masked_act_mul_and_blockwise_quant(gu, cnt))
    else:
        g, out = _graph(lambda: hpc.masked_act_mul_and_quant(gu, sc, cnt))
    n = sa.make_inputs(E, T, C, seed=10, device="cuda")
    gu.copy_(n["gate_up"])
    cnt.copy_(torch.tensor([T, 3, 0, 60, 1, T, 17, 2], dtype=torch.int32))
    sc.fill_(0.3)
    outs = out if blockwise else (out,)
    for o in outs:
        o.view(torch.uint8).fill_(0x5A)
    keep_before = [o.clone() for o in outs]
    g.replay()
    if blockwise:
        ref = hpc.masked_act_mul_and_blockwise_quant(gu, cnt, output=keep_before[0].clone(),
                                                     output_scale=keep_before[1].clone())
    else:
        ref = (hpc.masked_act_mul_and_quant(gu, sc, cnt, output=keep_before[0].clone()),)
    torch.cuda.synchronize()
    for a, b in zip(outs, ref):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))
    res = oact.masked_check(outs[0], outs[1] if blockwise else None, gu, cnt, T,
                            keep_before, scale=sc)
    assert oact.masked_ok(res), res


# ---- unsupported inputs ----------------------------------------------------------------------------
def test_unsupported_inputs_raise(hpc):
    w = lambda h: torch.ones(h, dtype=torch.bfloat16, device="cuda")  # noqa: E731
    sc = torch.ones(2, device="cuda")
    for h in (12, 16392):
        with pytest.raises(RuntimeError):
            hpc.fused_rmsnorm_with_scale(torch.ones(2, h, dtype=torch.bfloat16, device="cuda"), w(h),
                                         scale=sc)
    with pytest.raises(RuntimeError):
        hpc.fused_rmsnorm_with_scale(torch.ones(2, 64, device="cuda"), w(64), scale=sc)
    with pytest.raises(RuntimeError):
        hpc.fused_rmsnorm_with_scale(torch.ones(2, 64, dtype=torch.bfloat16, device="cuda"), w(64),
                                     scale=sc[:1], is_moe=True)
    gu = torch.ones(12, 2 * 256, dtype=torch.bfloat16, device="cuda")
    cnt = torch.ones(5, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match="multiple of the number of experts"):
        hpc.masked_act_mul_and_quant(gu, sc[:1], cnt)
    cnt = torch.ones(4, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match="multiple of 128"):
        hpc.masked_act_mul_and_blockwise_quant(gu[:, :192].contiguous(), cnt)
    with pytest.raises(RuntimeError, match="output must be"):
        hpc.masked_act_mul_and_quant(gu, sc[:1], cnt, output=torch.empty(12, 256, device="cuda"))
    with pytest.raises(RuntimeError, match="output_scale must be"):
        hpc.masked_act_mul_and_blockwise_quant(gu, cnt, output_scale=torch.empty(2, 12, device="cuda"))
