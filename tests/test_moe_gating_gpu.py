"""MoE top-k gating on the GPU against the fp64 oracle (oracle/moe_gating.py): ids exactly, weights
within the oracle's bound, planted ties to the lower id; column-slice views, caller outputs, NaN and
-inf rows, CUDA-graph replay, and the route GEMM -> gating -> blockwise FusedMoE chain."""
import numpy as np
import pytest
import torch

from oracle import gemm as ogm
from oracle import moe as om
from oracle import moe_gating as og
from synth import moe as sm
from synth import moe_gating as sg

pytestmark = pytest.mark.gpu

TOKENS = [1, 7, 128, 4097, 65536]
SPREAD = 1024  # rows the oracle checks at the largest T


def _dtype(dt):
    return torch.float32 if dt == "fp32" else torch.bfloat16


def _run(hpc, c, **kw):
    logits = c["store"].cuda()[:, :c["cfg"]["E"]]
    bias = None if c["bias"] is None else c["bias"].cuda()
    ids, w = hpc.moe_topk_gating(logits, **{**sg.hpc_kwargs(c["cfg"], bias), **kw})
    torch.cuda.synchronize()
    return ids.cpu(), w.cpu()


def _check(c, ids, w, rows=None):
    x = c["x"] if rows is None else c["x"][rows]
    ref = sg.oracle(x, c["cfg"], c["bias"])
    res = og.check(ids, w, ref, rows)
    assert not og.failed(res), res
    return ref


@pytest.mark.parametrize("T", TOKENS)
@pytest.mark.parametrize("dt", ["fp32", "bf16"])
@pytest.mark.parametrize("name", list(sg.CONFIGS))
def test_gating_matches_oracle(hpc, name, dt, T):
    cfg = sg.CONFIGS[name]
    rows = np.linspace(0, T - 1, SPREAD).astype(np.int64) if T > SPREAD * 8 else None
    pad = 8 if T % 2 == 0 else 0  # even T: rows of a wider buffer
    c = sg.make_case(cfg, T, _dtype(dt), seed=sg.seed_of(name, dt, T), pad=pad, rows=rows)
    ids, w = _run(hpc, c)
    assert ids.shape == (T, cfg["topk"]) and w.shape == (T, cfg["topk"])
    _check(c, ids, w, rows)


@pytest.mark.parametrize("dt", ["fp32", "bf16"])
@pytest.mark.parametrize("name", list(sg.CONFIGS))
def test_planted_ties_go_to_lower_id(hpc, name, dt):
    c = sg.make_case(sg.CONFIGS[name], 128, _dtype(dt), seed=sg.seed_of(name, dt, "ties"),
                     kind="ties", pad=8)
    ids, w = _run(hpc, c)
    _check(c, ids, w)
    gs = c["cfg"]["E"] // c["cfg"]["G"]
    assert len(c["planted"]) >= 100
    for t, lo, hi, what in c["planted"]:
        got = set(ids[t].tolist())
        if what == "expert":
            assert lo in got and hi not in got, (t, lo, hi, ids[t])
        else:  # the lower group is chosen: some of its experts may be picked, none of the other's
            assert not any(hi * gs <= e < (hi + 1) * gs for e in got), (t, lo, hi, ids[t])


@pytest.mark.parametrize("dt", ["fp32", "bf16"])
@pytest.mark.parametrize("name", list(sg.CONFIGS) + ["odd"])
def test_nan_and_inf_rows(hpc, name, dt):
    cfg = sg.ODD if name == "odd" else sg.CONFIGS[name]
    c = sg.special_rows(cfg, _dtype(dt), seed=sg.seed_of(name, dt, "special"),
                        pad=3 if name == "odd" else 8)
    ids, w = _run(hpc, c)
    _check(c, ids, w)  # distinct, in range, and equal to the oracle's total order
    ref = sg.oracle(c["x"], cfg, c["bias"])
    for t in range(3, 8):  # -inf keys are never chosen while finite ones are available
        if cfg["scoring"] == 0 and c["bias"] is None:
            assert np.isfinite(c["x"][t, ids[t].numpy()]).all()
    assert np.array_equal(ids.numpy(), ref["ids"])


@pytest.mark.parametrize("dt", ["fp32", "bf16"])
def test_column_slice_equals_contiguous_copy(hpc, dt):
    cfg = sg.CONFIGS["deepseek_v2"]
    full = sg.random_logits(300, 192, _dtype(dt), seed=5, device="cuda", width=192)
    view = full[:, :160]
    a = hpc.moe_topk_gating(view, **sg.hpc_kwargs(cfg, None))
    b = hpc.moe_topk_gating(view.contiguous(), **sg.hpc_kwargs(cfg, None))
    assert view.stride(0) == 192
    assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))


def test_caller_outputs_written_in_place(hpc):
    cfg = sg.CONFIGS["deepseek_v3"]
    x = sg.random_logits(33, 256, seed=6, device="cuda")
    bias = torch.randn(256, device="cuda") * 0.1
    ids = torch.full((33, 8), -7, dtype=torch.int32, device="cuda")
    w = torch.full((33, 8), -7.0, device="cuda")
    r = hpc.moe_topk_gating(x, **sg.hpc_kwargs(cfg, bias), topk_ids=ids, topk_weights=w)
    assert r[0].data_ptr() == ids.data_ptr() and r[1].data_ptr() == w.data_ptr()
    fresh = hpc.moe_topk_gating(x, **sg.hpc_kwargs(cfg, bias))
    assert torch.equal(ids, fresh[0]) and torch.equal(w, fresh[1])
    e = hpc.moe_topk_gating(x[:0], **sg.hpc_kwargs(cfg, bias))
    assert e[0].shape == (0, 8) and e[1].shape == (0, 8)


@pytest.mark.parametrize("name", ["qwen3", "deepseek_v3"])
def test_graph_replay_matches_eager(hpc, name):
    cfg = sg.CONFIGS[name]
    bias = torch.randn(cfg["E"], device="cuda") * 0.1 if cfg["bias"] else None
    kw = sg.hpc_kwargs(cfg, bias)
    static = sg.random_logits(512, cfg["E"], seed=1, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        hpc.moe_topk_gating(static, **kw)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = hpc.moe_topk_gating(static, **kw)
    for seed in (2, 3, 4):
        static.copy_(sg.random_logits(512, cfg["E"], seed=seed, device="cuda"))
        g.replay()
        ref = hpc.moe_topk_gating(static.clone(), **kw)
        torch.cuda.synchronize()
        assert torch.equal(out[0], ref[0])
        assert torch.equal(out[1].view(torch.int32), ref[1].view(torch.int32))


def test_route_gemm_gating_fused_moe_chain_in_one_graph(hpc):
    """gemm_bf16xfp32 (fp32 out, 128 columns of which 96 are experts) -> moe_topk_gating on the
    column slice -> fuse_moe_blockwise_fp8, captured as one graph; each stage checked from the
    kernel's own input to it."""
    from test_moe_gpu import _close

    T, K, N, E, k, H, I = 96, 512, 128, 96, 6, 512, 256
    cfg = dict(E=E, topk=k, scoring=0, renormalize=False, bias=False, G=8, topk_group=3,
               factor=1.0)
    xr, _, w_high, w_low, scale = ogm.make_inputs(T, N, K, seed=11)
    d = sm.make_moe_blockwise_routed_inputs(T, k, H, I, E, seed=12)
    c = {n: (v.cuda() if isinstance(v, torch.Tensor) else v) for n, v in d.items()}
    xg, wh, wl = xr.cuda(), w_high.cuda(), w_low.cuda()

    def chain():
        logits = hpc.gemm_bf16xfp32(xg, wh, wl, scale, use_fp32_output=True)
        ids, w = hpc.moe_topk_gating(logits[:, :E], **sg.hpc_kwargs(cfg, None))
        y = hpc.fuse_moe_blockwise_fp8(c["x"], c["x_scale"], c["gate_up_weight"],
                                       c["gate_up_weight_scale"], c["down_weight"],
                                       c["down_weight_scale"], ids, w, 0, E)
        return logits, ids, w, y

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        chain()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        logits, ids, w, y = chain()
    g.replay()
    torch.cuda.synchronize()
    exact = ogm.gemm_split_exact(xr, w_high, w_low, scale)
    rel = (logits.cpu().double() - exact).norm() / exact.norm()
    assert rel < 1e-5, rel
    lg = logits[:, :E].cpu()
    ref = sg.oracle(lg, cfg, None)
    res = og.check(ids.cpu(), w.cpu(), ref)
    assert not og.failed(res), res
    gt = om.fuse_moe_blockwise(d["x"], d["x_scale"], d["gate_up_weight"], d["gate_up_weight_scale"],
                               d["down_weight"], d["down_weight_scale"], ids.cpu(), w.cpu(), 0,
                               None)
    _close(y, gt, 0.01, 0.01, "gemm -> gating -> moe blockwise", outlier_ppm=5, outlier_cap=0.05)


def test_rejected_arguments_raise(hpc):
    x = torch.zeros(4, 256, device="cuda")
    b = torch.zeros(256, device="cuda")
    for kw in (dict(topk=0), dict(topk=17), dict(num_expert_group=3),
               dict(num_expert_group=8, topk_group=9), dict(num_expert_group=64, topk=8),
               dict(correction_bias=b, num_expert_group=256, topk_group=8),
               dict(correction_bias=b[:255]), dict(scoring=2),
               dict(topk_ids=torch.zeros(4, 8, dtype=torch.int64, device="cuda"))):
        with pytest.raises(RuntimeError):
            hpc.moe_topk_gating(x, **{"topk": 8, **kw})
    for bad in (torch.zeros(4, 520, device="cuda"), torch.zeros(4, 258, device="cuda")[:, :256],
                torch.zeros(4, 260, device="cuda")[:, 1:257], x.half(), x.t()):
        with pytest.raises(RuntimeError):
            hpc.moe_topk_gating(bad, 8)
