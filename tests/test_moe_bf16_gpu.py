"""hpc.fuse_moe_bf16 and hpc.group_gemm_bf16 checked stage by stage against oracle/moe_bf16.py.

Every scratch buffer is filled with a sentinel first (NaN for bf16, -7 for ints), so a stage that
leaves an element it owns unwritten, or reads one it should not, shows up whatever the allocator
handed out. The public op must give the staged launch's bits. Shapes: a small one, Qwen3-30B-A3B-,
DeepSeek-V2-Lite- (I = 1408: an odd number of 128-column blocks) and Mixtral-like experts, H = 640
(a ragged 256-column Down tile) and the 512-local-expert limit; token counts 1, 3, 64 and ~1000."""
import pytest
import torch

from oracle import moe_bf16 as ob, moe_exact as ox
from synth.moe_bf16 import make_group_gemm_bf16_inputs, make_moe_bf16_inputs

pytestmark = pytest.mark.gpu

SENTINEL = {torch.bfloat16: float("nan"), torch.int32: -7}


def _cuda(d):
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in d.items()}


def _args(c):
    return (c["x"], c["gate_up_weight"], c["down_weight"], c["topk_ids"], c["topk_scale"],
            c["shared_output"], c["rank_ep"], c["num_expert_total"])


def _run_staged(hpc, c, output=None):
    from hpc.fuse_moe import _bf16_scratch, _launch_bf16

    s = _bf16_scratch(c["x"], c["gate_up_weight"], c["topk_ids"])
    for t in s.values():
        t.fill_(SENTINEL[t.dtype])
    y = torch.full(c["x"].shape, float("nan"), dtype=torch.bfloat16, device="cuda")
    _launch_bf16(y, *_args(c), s)
    if output is not None:
        output.fill_(float("nan"))
    public = hpc.fuse_moe_bf16(c["x"], c["gate_up_weight"], c["down_weight"], c["topk_ids"],
                               c["topk_scale"], c["rank_ep"], c["num_expert_total"],
                               shared_output=c["shared_output"], output=output)
    torch.cuda.synchronize()
    if output is not None:
        assert public.data_ptr() == output.data_ptr(), "caller-given output not returned"
    assert torch.equal(public.view(torch.int16), y.view(torch.int16)), \
        "public op differs from the staged launch"
    return y.cpu(), {k: v.cpu() for k, v in s.items()}


def _check_all(hpc, d, tag, seed=0, output=None):
    c = _cuda(d)
    y, s = _run_staged(hpc, c, output)
    E = d["gate_up_weight"].size(0)
    r = ob.route(d["topk_ids"], E, d["rank_ep"], d["num_expert_total"])
    ob.check_route(r, d["x"], s)
    rows = ob.rows_to_check(r, seed=seed)
    st = dict(rows=int(r["src_token"].numel()), checked=int(rows.numel()), flips=0, explained=0,
              down=0.0, down_acc=0.0)
    if rows.numel():
        g = ob.check_gateup(s["gate_up_input"], r, d["gate_up_weight"], rows, s["down_input"])
        st.update(g)
        yd, B = ob.down_exact(s["down_input"], r, d["down_weight"], rows)
        st["down"] = ox.check_down(s["down_output"][rows], yd, B, tag=f"{tag} down")
        st["down_acc"] = ox.accumulation_probe(s["down_output"][rows], yd, B, tag=f"{tag} down")
    o, B = ox.reduce_exact(s["down_output"], s["topk_pos"], d["topk_scale"], d["shared_output"])
    st["reduce"] = ox.check_down(y, o, B, tag=f"{tag} reduce")
    st["reduce_acc"] = ox.accumulation_probe(y, o, B, tag=f"{tag} reduce")
    print(f"\n[{tag}] rows {st['rows']} checked {st['checked']} flips {st['flips']} (explained "
          f"{st['explained']}) down err/B {st['down']:.3f} acc/E>={st['down_acc']:.3f} reduce err/B "
          f"{st['reduce']:.3f} acc/E>={st['reduce_acc']:.3f}")
    return st, c


# (name, E_total, k, H, I)
SMALL = ("small", 8, 2, 512, 256)
QWEN = ("qwen3_30b_a3b", 128, 8, 2048, 768)
DSV2L = ("deepseek_v2_lite", 64, 6, 2048, 1408)
MIXTRAL = ("mixtral", 8, 2, 4096, 14336)
RAGGED = ("h640", 16, 4, 640, 256)


@pytest.mark.parametrize("shape", [SMALL, QWEN, DSV2L, RAGGED], ids=lambda s: s[0])
@pytest.mark.parametrize("T", [1, 3, 64, 1000])
def test_stages_uniform(hpc, shape, T):
    name, E, k, H, I = shape
    d = make_moe_bf16_inputs(T, k, H, I, E, seed=T * 7 + H)
    _check_all(hpc, d, f"{name} T{T}", seed=T)


@pytest.mark.parametrize("T", [1, 3, 64])
def test_stages_mixtral_small_batch(hpc, T):
    name, E, k, H, I = MIXTRAL
    d = make_moe_bf16_inputs(T, k, H, I, E, seed=T + 5)
    _check_all(hpc, d, f"{name} T{T}", seed=T)


@pytest.mark.parametrize("routing", ["hot", "sparse"])
def test_stages_routing(hpc, routing):
    name, E, k, H, I = QWEN
    T = 16 if routing == "sparse" else 1000
    d = make_moe_bf16_inputs(T, k, H, I, E, routing=routing, seed=11)
    st, _ = _check_all(hpc, d, f"{name} {routing} T{T}")
    if routing == "hot":
        assert st["rows"] == T * k


@pytest.mark.parametrize("rank_ep", [1, 3])
def test_stages_other_rank(hpc, rank_ep):
    """EP size 4: a quarter of the experts are local; some tokens have none of theirs here."""
    d = make_moe_bf16_inputs(300, 2, 512, 256, 32, routing="other_rank", size_ep=4,
                             rank_ep=rank_ep, shared=True, seed=20 + rank_ep)
    st, _ = _check_all(hpc, d, f"ep4 rank {rank_ep}")
    assert 0 < st["rows"] < 300 * 2


def test_stages_512_local_experts(hpc):
    d = make_moe_bf16_inputs(256, 8, 256, 128, 512, seed=13)
    _check_all(hpc, d, "512 experts")


def test_shared_output_and_given_output(hpc):
    d = make_moe_bf16_inputs(64, 2, 512, 256, 8, shared=True, seed=14)
    out = torch.empty((64, 512), dtype=torch.bfloat16, device="cuda")
    _check_all(hpc, d, "shared + output", output=out)


def test_two_calls_bit_identical(hpc):
    c = _cuda(make_moe_bf16_inputs(1000, 8, 2048, 768, 128, seed=15))
    a = hpc.fuse_moe_bf16(*_args(c)[:5], c["rank_ep"], c["num_expert_total"])
    b = hpc.fuse_moe_bf16(*_args(c)[:5], c["rank_ep"], c["num_expert_total"])
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_zero_tokens(hpc):
    c = _cuda(make_moe_bf16_inputs(0, 2, 256, 128, 8, seed=16))
    y = hpc.fuse_moe_bf16(*_args(c)[:5], 0, 8)
    assert y.shape == (0, 256)


@pytest.mark.parametrize("seqlens,n,k", [([0, 200, 0, 1, 129, 0], 384, 512),
                                         ([5, 0, 0, 300], 640, 256),
                                         ([0, 0, 0], 256, 128)])
def test_group_gemm_bf16(hpc, seqlens, n, k):
    """Empty groups, a ragged 256-column tile (n = 384, 640), and rows outside every group (left
    unwritten)."""
    d = make_group_gemm_bf16_inputs(seqlens, n, k)
    c = _cuda(d)
    out = torch.full((d["x"].size(0), n), float("nan"), dtype=torch.bfloat16, device="cuda")
    y = hpc.group_gemm_bf16(c["x"], c["weight"], c["seqlens"], c["cu_seqlens"], output=out)
    torch.cuda.synchronize()
    assert y.data_ptr() == out.data_ptr()
    want, B = ob.group_gemm_exact(d["x"], d["weight"], d["seqlens"], d["cu_seqlens"])
    yc = y.cpu()
    inside = ~torch.isnan(want[:, 0])
    assert torch.isnan(yc[~inside].float()).all(), "rows outside every group were written"
    if inside.any():
        ox.check_down(yc[inside], want[inside], B[inside], tag="group_gemm_bf16")
        ox.accumulation_probe(yc[inside], want[inside], B[inside], tag="group_gemm_bf16")


def test_gating_chain(hpc):
    """moe_topk_gating -> fuse_moe_bf16 on one stream, against the chain's own topk outputs."""
    name, E, k, H, I = QWEN
    d = make_moe_bf16_inputs(200, k, H, I, E, seed=17)
    c = _cuda(d)
    logits = torch.randn((200, E), generator=torch.Generator().manual_seed(3)).cuda()
    ids, w = hpc.moe_topk_gating(logits, k)
    c.update(topk_ids=ids, topk_scale=w)
    torch.cuda.synchronize()
    d.update(topk_ids=ids.cpu(), topk_scale=w.cpu())
    st, _ = _check_all(hpc, d, "gating chain")
    assert st["rows"] == 200 * k


def _capture(fn):
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()  # warm-up: scheduler counters and smem attributes set up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        out = fn()
    return g, out


def _refill(dst, src):
    for key in ("x", "topk_ids", "topk_scale"):
        dst[key].copy_(src[key])


def test_graph_replay_on_new_data(hpc):
    name, E, k, H, I = QWEN
    d0 = make_moe_bf16_inputs(64, k, H, I, E, seed=18)
    d1 = make_moe_bf16_inputs(64, k, H, I, E, seed=19)
    d1["gate_up_weight"], d1["down_weight"] = d0["gate_up_weight"], d0["down_weight"]
    c = _cuda(d0)
    g, out = _capture(lambda: hpc.fuse_moe_bf16(*_args(c)[:5], 0, E))
    c1 = _cuda(d1)
    _refill(c, c1)
    g.replay()
    torch.cuda.synchronize()
    eager = hpc.fuse_moe_bf16(*_args(c1)[:5], 0, E)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), eager.view(torch.int16))
    del g


def test_two_graphs_on_two_streams(hpc):
    name, E, k, H, I = QWEN
    ds = [make_moe_bf16_inputs(300, k, H, I, E, seed=30 + i) for i in range(2)]
    cs = [_cuda(d) for d in ds]
    graphs = [_capture(lambda c=c: hpc.fuse_moe_bf16(*_args(c)[:5], 0, E)) for c in cs]
    eager = [hpc.fuse_moe_bf16(*_args(c)[:5], 0, E) for c in cs]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for _ in range(3):
        for (g, _), s in zip(graphs, streams):
            with torch.cuda.stream(s):
                g.replay()
    torch.cuda.synchronize()
    for (_, out), e in zip(graphs, eager):
        assert torch.equal(out.view(torch.int16), e.view(torch.int16))
    del graphs
