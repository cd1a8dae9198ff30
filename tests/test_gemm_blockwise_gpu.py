"""hpc.blockwise_fp8_quant held bit for bit to oracle/gemm_blockwise.py's restatement, and
hpc.gemm_blockwise_fp8 held element by element to its fp64 oracle, on the synthetic inputs of
synth/gemm_blockwise.py and on the projection shapes of DeepSeek-V3 and Qwen3.

Each graded GEMM run prints `GEMM <tag> split=<s> worst_err/B=... acc/E>=...` (pytest -s)."""
import pytest
import torch

from oracle import gemm_blockwise as ob
from synth import gemm_blockwise as sb

pytestmark = pytest.mark.gpu

# (N, K) of real projections
SHAPES = {
    "dsv3_q_a_kv_a": (2112, 7168), "dsv3_kv_a": (576, 7168), "dsv3_q_a": (1536, 7168),
    "dsv3_q_b": (24576, 1536), "dsv3_kv_b": (32768, 512), "dsv3_o": (7168, 16384),
    "dsv3_shared_gate_up": (4096, 7168), "dsv3_shared_down": (7168, 2048),
    "qwen3_32b_gate_up": (10240, 5120), "qwen3_32b_o": (5120, 8192),
    "qwen3_32b_down": (5120, 25600),
    "qwen3_8b_qkv": (6144, 4096), "qwen3_8b_gate_up": (24576, 4096),
}
MS = (1, 8, 64, 256, 1024, 4096)


def _split(hpc, m, n, k):
    return hpc._ffi.lib.hpc_gemm_blockwise_fp8_config(m, n, k)


def _grade(hpc, x, xs, w, ws, rows, tag, out=None):
    m, k = x.shape
    n = w.size(0)
    split = _split(hpc, m, n, k)
    y = hpc.gemm_blockwise_fp8(x.cuda(), xs.cuda(), w.cuda(), ws.cuda(), out)
    assert y.shape == (m, n) and y.dtype == torch.bfloat16
    ye, B, _ = ob.gemm_exact(x, xs, w, ws, split, rows)
    worst, acc = ob.check(y[rows.cuda()].cpu(), ye, B, tag)
    print(f"GEMM {tag} split={split} worst_err/B={worst:.3g} acc/E>={acc:.3g}")
    return y


# ------------------------------------------------------------------------------------------------
# quantiser
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", (128, 640, 2048, 7168, 16384))
@pytest.mark.parametrize("m", (1, 3, 64, 1000, 4096))
def test_quant_bit_exact(hpc, m, k):
    x = sb.quant_input(m, k, seed=m * 7 + k)
    q, sc = hpc.blockwise_fp8_quant(x.cuda())
    assert q.dtype == torch.float8_e4m3fn and q.shape == (m, k) and q.is_contiguous()
    assert sc.dtype == torch.float32 and sc.shape == (m, k // 128) and sc.is_contiguous()
    wq, ws = ob.quant(x)
    assert ob.quant_mismatch(q.cpu(), sc.cpu(), wq, ws) == (0, 0)


def test_quant_strided_input_and_given_outputs(hpc):
    m, k = 1000, 2048
    xc = sb.quant_input(m, k, seed=5, ld=k + 72)
    x = torch.empty((m, k + 72), dtype=torch.bfloat16, device="cuda")[:, :k]
    x.copy_(xc)
    assert not x.is_contiguous() and x.stride(0) == k + 72
    q0 = torch.full((m, k), 0x7F, dtype=torch.uint8, device="cuda").view(torch.float8_e4m3fn)
    s0 = torch.full((m, k // 128), float("nan"), device="cuda")
    q, sc = hpc.blockwise_fp8_quant(x, q0, s0)
    assert q.data_ptr() == q0.data_ptr() and sc.data_ptr() == s0.data_ptr()
    wq, ws = ob.quant(x.cpu())
    assert ob.quant_mismatch(q.cpu(), sc.cpu(), wq, ws) == (0, 0)


def test_quant_rejects_bad_outputs(hpc):
    x = torch.zeros((4, 256), dtype=torch.bfloat16, device="cuda")
    bad = [(torch.empty((4, 256), dtype=torch.uint8, device="cuda"), None),
           (torch.empty((4, 128), dtype=torch.float8_e4m3fn, device="cuda"), None),
           (torch.empty((4, 256), dtype=torch.float8_e4m3fn), None),
           (None, torch.empty((2, 4), device="cuda").t()),
           (None, torch.empty((4, 2), dtype=torch.float16, device="cuda"))]
    for o, s in bad:
        with pytest.raises(RuntimeError, match="blockwise_fp8_quant"):
            hpc.blockwise_fp8_quant(x, o, s)
    with pytest.raises(RuntimeError, match="multiple of 128"):
        hpc.blockwise_fp8_quant(torch.zeros((4, 200), dtype=torch.bfloat16, device="cuda"))
    q, sc = hpc.blockwise_fp8_quant(x[:0])
    assert q.shape == (0, 256) and sc.shape == (0, 2)


def test_quant_output_feeds_fuse_moe_blockwise(hpc):
    """The (x, x_scale) pair goes into fuse_moe_blockwise_fp8 as is, and the result equals the
    same call with x_scale built by torch ops from the oracle's codes."""
    T, H, I, E, K = 64, 512, 256, 8, 2
    x = sb.quant_input(T, H, seed=9).float().clamp(-4, 4).to(torch.bfloat16).cuda()
    q, sc = hpc.blockwise_fp8_quant(x)
    g = torch.Generator().manual_seed(1)
    guw = (torch.randn((E, 2 * I, H), generator=g) * 0.1).to(torch.float8_e4m3fn).cuda()
    dw = (torch.randn((E, H, I), generator=g) * 0.1).to(torch.float8_e4m3fn).cuda()
    guws = torch.rand((E, 2 * I // 128, H // 128), generator=g).cuda() + 0.5
    dws = torch.rand((E, H // 128, 4), generator=g).cuda() + 0.5  # K blocks padded to 4
    ids = torch.stack([torch.randperm(E, generator=g)[:K] for _ in range(T)]).int().cuda()
    ts = torch.rand((T, K), generator=g).cuda()
    y = hpc.fuse_moe_blockwise_fp8(q, sc, guw, guws, dw, dws, ids, ts, 0, E)
    wq, ws = ob.quant(x.cpu())
    y2 = hpc.fuse_moe_blockwise_fp8(wq.cuda(), ws.cuda(), guw, guws, dw, dws, ids, ts, 0, E)
    torch.cuda.synchronize()
    assert y.shape == (T, H) and torch.isfinite(y.float()).all()
    assert torch.equal(y.view(torch.int16), y2.view(torch.int16))


# ------------------------------------------------------------------------------------------------
# GEMM
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ci", range(len(sb.CASES)), ids=[sb.tag(c) for c in sb.CASES])
def test_gemm_synthetic(hpc, ci):
    c = sb.CASES[ci]
    d = sb.make_inputs(c)
    rows = torch.unique(torch.cat([ob.rows_to_check(c["m"], c["n"], c["k"]), d["cancel_rows"]]))
    _grade(hpc, d["x"], d["xs"], d["w"], d["ws"], rows, sb.tag(c))


@pytest.mark.parametrize("m", MS)
@pytest.mark.parametrize("name", list(SHAPES))
def test_gemm_projection_shapes(hpc, name, m):
    n, k = SHAPES[name]
    x, xs, w, ws = sb.real_inputs(m, n, k, seed=m)
    # large shapes: both sides of every 128-row tile boundary, first and last rows and a sample
    rows = ob.rows_to_check(m, n, k, n_random=4, small=1 << 24, tile_m=128)
    _grade(hpc, x, xs, w, ws, rows, f"{name}_m{m}")


def test_shapes_reach_every_split(hpc):
    got = {_split(hpc, m, n, k) for n, k in SHAPES.values() for m in MS}
    got |= {_split(hpc, c["m"], c["n"], c["k"]) for c in sb.CASES}
    assert got == {1, 2, 4, 8}, got


# ------------------------------------------------------------------------------------------------
# plumbing
# ------------------------------------------------------------------------------------------------
def test_nan_output_overwritten_and_calls_identical(hpc):
    for c in sb.CASES:
        d = {k: v.cuda() for k, v in sb.make_inputs(c).items()}
        out = torch.full((c["m"], c["n"]), float("nan"), dtype=torch.bfloat16, device="cuda")
        y = hpc.gemm_blockwise_fp8(d["x"], d["xs"], d["w"], d["ws"], out)
        assert y.data_ptr() == out.data_ptr()
        assert torch.isfinite(out.float()).all(), sb.tag(c)
        y2 = hpc.gemm_blockwise_fp8(d["x"], d["xs"], d["w"], d["ws"])
        assert torch.equal(out.view(torch.int16), y2.view(torch.int16)), sb.tag(c)


def test_m_zero_and_bad_arguments(hpc):
    w = torch.zeros((256, 512), dtype=torch.float8_e4m3fn, device="cuda")
    ws = torch.ones((2, 4), device="cuda")
    x = torch.zeros((0, 512), dtype=torch.float8_e4m3fn, device="cuda")
    y = hpc.gemm_blockwise_fp8(x, torch.ones((0, 4), device="cuda"), w, ws)
    assert y.shape == (0, 256)
    x = torch.zeros((4, 512), dtype=torch.float8_e4m3fn, device="cuda")
    xs = torch.ones((4, 4), device="cuda")
    with pytest.raises(RuntimeError, match="weight_scale"):
        hpc.gemm_blockwise_fp8(x, xs, w, torch.ones((2, 5), device="cuda"))
    with pytest.raises(RuntimeError, match="x_scale"):
        hpc.gemm_blockwise_fp8(x, xs.t().contiguous().t(), w, ws)
    with pytest.raises(RuntimeError, match="N"):
        hpc.gemm_blockwise_fp8(x, xs, w[:100], ws)


def _quant_gemm(hpc, a, w, ws):
    q, sc = hpc.blockwise_fp8_quant(a)
    return hpc.gemm_blockwise_fp8(q, sc, w, ws)


@pytest.mark.parametrize("m,n,k", [(8, 2112, 7168), (1024, 4096, 2048)])
def test_graph_replay_equals_eager_on_two_streams(hpc, m, n, k):
    _, _, w, ws = sb.real_inputs(1, n, k, seed=3)
    w, ws = w.cuda(), ws.cuda()
    g = torch.Generator().manual_seed(4)
    inputs = [torch.randn((m, k), generator=g).to(torch.bfloat16).cuda() for _ in range(4)]
    a = [torch.empty_like(inputs[0]) for _ in range(2)]
    graphs, outs = [], []
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for i in range(2):
            a[i].copy_(inputs[i])
            _quant_gemm(hpc, a[i], w, ws)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    for i in range(2):
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            outs.append(_quant_gemm(hpc, a[i], w, ws))
        graphs.append(gr)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for i in range(2):
        a[i].copy_(inputs[2 + i])
    torch.cuda.synchronize()
    for i in range(2):
        with torch.cuda.stream(streams[i]):
            graphs[i].replay()
    torch.cuda.synchronize()
    for i in range(2):
        want = _quant_gemm(hpc, inputs[2 + i], w, ws)
        torch.cuda.synchronize()
        assert torch.equal(outs[i].view(torch.int16), want.view(torch.int16)), i
