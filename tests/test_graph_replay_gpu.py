"""The persistent kernels under CUDA-graph capture and replay, the way serving code runs them.

The grouped GEMM (behind both FusedMoE pipelines) and the block-sparse prefill claim their work from
a device-side counter that the last CTA of each launch re-arms. These tests check that
  a. a process whose first call of an op is made inside `torch.cuda.graph` captures and replays it;
  b. a graph replayed on new data (routing, kv lengths, masks copied into its static inputs) gives
     exactly what an eager call on the same data gives;
  c. graphs captured on torch's shared default capture stream and replayed concurrently on two
     streams each give the eager result, and eager calls afterwards are still right;
  d. 200 distinct streams, all running at once, each get a working scheduler.
Bit equality is the criterion: every op here is deterministic (checked per op first), so any
difference is a scheduling error, not rounding."""
import ctypes
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
REPO = Path(__file__).resolve().parents[1]


def _bits(t):
    """Byte view for comparisons that also match NaN rows (a fully masked prefill Q tile is NaN)."""
    return t.contiguous().view(torch.uint8)


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


# ------------------------------------------------------------------------------------------------
# Cases: make(seed) builds a full input dict on the GPU, `data` names the tensors that change
# between replays (copied into the graph's static inputs), run(d) calls the op.
# ------------------------------------------------------------------------------------------------
class _MoeBlockwise:
    data = ("x", "x_scale", "topk_ids", "topk_scale")

    def __init__(self, T=256, H=512, I=256, E=64):
        self.shape = (T, H, I, E)

    def make(self, seed):
        from synth.moe import make_moe_blockwise_inputs

        T, H, I, E = self.shape
        d = make_moe_blockwise_inputs(T, 8, H, I, E, seed=seed, device="cuda")
        # more rows for the first experts in odd seeds: the routing (and every expert's tile
        # count) differs from replay to replay
        if seed % 2:
            d["topk_ids"][:, 0] = torch.randint(0, 4, (T,), device="cuda", dtype=torch.int32,
                                                generator=torch.Generator("cuda").manual_seed(seed))
            d["topk_ids"], _ = torch.sort(d["topk_ids"], dim=1)
        return d

    def run(self, hpc, d):
        E = self.shape[3]
        return hpc.fuse_moe_blockwise(d["x"], d["x_scale"], d["gate_up_weight"],
                                      d["gate_up_weight_scale"], d["down_weight"],
                                      d["down_weight_scale"], d["topk_ids"], d["topk_scale"], 0, E)


class _MoePertensor:
    data = ("x", "topk_ids", "topk_scale")

    def __init__(self, T=300, H=512, I=256, E=32):
        self.shape = (T, H, I, E)

    def make(self, seed):
        from synth.moe import make_moe_pertensor_inputs

        T, H, I, E = self.shape
        d = make_moe_pertensor_inputs(T, 8, H, I, E, routing="uniform" if seed % 2 == 0 else "repeat",
                                      seed=seed)
        return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in d.items()}

    def run(self, hpc, d):
        return hpc.fuse_moe(d["x"], d["gate_up_weight"], d["down_weight"], d["gate_up_scale"],
                            d["down_scale"], d["act_scale"], d["topk_ids"], d["topk_scale"], 0,
                            self.shape[3])


def _partition(m, groups, gen):
    """Random split of m rows over `groups` groups (some empty), as int32 seqlens and cu_seqlens."""
    cuts = torch.sort(torch.randint(0, m + 1, (groups - 1,), generator=gen)).values
    edges = torch.cat([torch.tensor([0]), cuts, torch.tensor([m])])
    seqlens = (edges[1:] - edges[:-1]).to(torch.int32)
    return seqlens, edges.to(torch.int32)


class _GemmBlockwise:
    data = ("x", "seqlens", "cu", "xs_t")
    G, M, N, K, AVG = 16, 1000, 512, 512, 62  # avg 62 -> 64-column scale granules

    def make(self, seed):
        g = torch.Generator().manual_seed(seed)
        seqlens, cu = _partition(self.M, self.G, g)
        x = torch.randn((self.M, self.K), generator=g).to(torch.float8_e4m3fn)
        w = torch.randn((self.G, self.N, self.K), generator=g).to(torch.float8_e4m3fn)
        ws = torch.rand((self.G, self.N // 128, (self.K // 128 + 3) // 4 * 4), generator=g) / 16
        xs_rows = torch.rand((self.M, self.K // 128), generator=g) + 0.5
        tile = 64
        xs_t = torch.zeros((self.K // 128, self.M + self.G * tile))
        col = 0
        for gi in range(self.G):
            r = int(seqlens[gi])
            xs_t[:, col:col + r] = xs_rows[int(cu[gi]):int(cu[gi]) + r].t()
            col += (r + tile - 1) // tile * tile
        return dict(x=x.cuda(), w=w.cuda(), seqlens=seqlens.cuda(), cu=cu.cuda(), xs_t=xs_t.cuda(),
                    ws=ws.cuda())

    def run(self, hpc, d):
        return hpc.group_gemm_blockwise_fp8(d["x"], d["w"], d["seqlens"], d["cu"], d["xs_t"],
                                            d["ws"], num_seq_per_group_avg=self.AVG)


class _GemmPertensor:
    data = ("x", "seqlens", "cu", "ys")
    G, M, N, K = 8, 1500, 1024, 1024

    def make(self, seed):
        g = torch.Generator().manual_seed(seed)
        seqlens, cu = _partition(self.M, self.G, g)
        x = torch.randn((self.M, self.K), generator=g).to(torch.float8_e4m3fn)
        w = torch.randn((self.G, self.N, self.K), generator=g).to(torch.float8_e4m3fn)
        ys = torch.rand((self.G,), generator=g) / 32
        return dict(x=x.cuda(), w=w.cuda(), seqlens=seqlens.cuda(), cu=cu.cuda(), ys=ys.cuda())

    def run(self, hpc, d):
        return hpc.group_gemm_pertensor_fp8(d["x"], d["w"], d["seqlens"], d["cu"], d["ys"],
                                            num_seq_per_group_avg=self.M // self.G)


class _Prefill:
    """Two requests, q_total query tokens in all (at most max_q each), kv capacity kv_cap each;
    replays move the query split, the kv lengths and the block mask."""
    data = ("q", "qscale", "cu_seqlens_q", "seqlens_kv", "block_mask")

    def __init__(self, kpt, q_total=812, max_q=512, kv_cap=1024, hq=8, hkv=2):
        self.kpt, self.q_total, self.max_q, self.kv_cap = kpt, q_total, max_q, kv_cap
        self.hq, self.hkv = hq, hkv

    def make(self, seed):
        from synth.prefill import make_inputs

        g = torch.Generator().manual_seed(seed)
        mq, qt = self.max_q, self.q_total
        a = mq if seed == 0 else int(torch.randint(qt - mq, mq + 1, (1,), generator=g))
        q_lens = [a, qt - a]
        d = make_inputs([mq, qt - mq], [self.kv_cap] * 2, self.hq, self.hkv, 0.3,
                        self.kpt, seed=seed, device="cuda")
        kv = [self.kv_cap if seed == 0 else int(torch.randint(ql, self.kv_cap + 1, (1,), generator=g))
              for ql in q_lens]
        d["cu_seqlens_q"] = torch.tensor([0, q_lens[0], self.q_total], dtype=torch.int32, device="cuda")
        d["seqlens_kv"] = torch.tensor(kv, dtype=torch.int32, device="cuda")
        d["block_mask"] = d["block_mask"].to(torch.uint8).contiguous()
        return d

    def run(self, hpc, d):
        qt = (hpc.QuantType.QPERTOKEN_PERHEAD_KPERTOKEN_PERHEAD_VPERHEAD if self.kpt
              else hpc.QuantType.QPERTOKEN_PERHEAD_KPERTENSOR_VPERTENSOR)
        return hpc.attention_with_kvcache_blocksparse_prefill_fp8(
            d["q"], d["kcache"], d["vcache"], d["qscale"], d["kscale"], d["vscale"],
            d["cu_seqlens_q"], d["block_ids"], d["seqlens_kv"], self.max_q, quant_type=qt,
            block_mask=d["block_mask"])


class _Decode:
    """One decode step: the task map is scheduled on the device from the kv lengths, then the
    attention kernel reads it. The task-map workspace is made before any capture (creating its
    template copies a header from the host). Replays change q and the kv lengths."""

    def __init__(self, fp8, B=12, cap=1500, hkv=2, hq=16):
        self.fp8, self.B, self.cap, self.hkv, self.hq = fp8, B, cap, hkv, hq
        self.data = ("q", "kv_lens_total") + (("q_scale",) if fp8 else ())
        self.tm = None

    def make(self, seed):
        from synth.decode import make_decode_bf16_inputs, make_decode_fp8_inputs

        mk = make_decode_fp8_inputs if self.fp8 else make_decode_bf16_inputs
        d = mk(self.B, 1, [self.cap] * self.B, self.hkv, self.hq, seed=seed, device="cuda")
        if seed:
            g = torch.Generator().manual_seed(seed)
            d["kv_lens_total"] = torch.randint(1, self.cap + 1, (self.B,), generator=g,
                                               dtype=torch.int32).cuda()
        return d

    def workspace(self, hpc):
        if self.tm is None:
            self.tm = hpc.get_attention_decode_task_workspace(self.B, self.cap, self.hkv, 64)
        return self.tm

    def run(self, hpc, d):
        tm = self.workspace(hpc)
        hpc.assign_attention_decode_task(d["kv_lens_total"], tm, self.hkv, 1, True, 64)
        if self.fp8:
            return hpc.attention_decode_fp8(d["q"], d["kvcache"][:, 0], d["kvcache"][:, 1],
                                            d["block_ids"], d["kv_lens_total"], d["q_scale"],
                                            d["k_scale"], d["v_scale"], mtp=0, new_kv_included=True,
                                            task_map=tm)
        return hpc.attention_decode_bf16(d["q"], d["kvcache"][:, 0], d["kvcache"][:, 1],
                                         d["block_ids"], d["kv_lens_total"], mtp=0,
                                         new_kv_included=True, task_map=tm)


CASES = {
    "fuse_moe_blockwise": _MoeBlockwise,
    "fuse_moe": _MoePertensor,
    "group_gemm_blockwise_fp8": _GemmBlockwise,
    "group_gemm_pertensor_fp8": _GemmPertensor,
    "prefill_kvpertensor": lambda: _Prefill(False),
    "prefill_kpertoken": lambda: _Prefill(True),
    "decode_fp8": lambda: _Decode(True),
    "decode_bf16": lambda: _Decode(False),
}


def _capture(fn):
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn()
    return g, out


# ------------------------------------------------------------------------------------------------
# a. the first call of the process is made inside a capture
# ------------------------------------------------------------------------------------------------
def _child(name):
    """Run in a fresh process: capture the op's very first call, replay, compare with eager."""
    import hpc

    case = CASES[name]()
    d = case.make(0)
    if isinstance(case, _Decode):
        case.workspace(hpc)
    torch.cuda.synchronize()
    g, out = _capture(lambda: case.run(hpc, d))
    g.replay()
    got = out.clone()
    ref = case.run(hpc, d)
    torch.cuda.synchronize()
    ok = _same(got, ref)
    assert ok, f"{name}: replay of a first-call capture differs from eager"
    print("child ok", name)


@pytest.mark.parametrize("name", list(CASES))
def test_first_call_inside_capture(hpc, name):
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([str(REPO), str(REPO / "hpc-ops_b200"),
                                         str(Path(__file__).resolve().parent),
                                         env.get("PYTHONPATH", "")])
    code = f"import test_graph_replay_gpu as t; t._child({name!r})"
    r = subprocess.run([sys.executable, "-c", code], cwd=str(REPO), env=env, capture_output=True,
                       text=True, timeout=300)
    ok = r.returncode == 0 and "child ok" in r.stdout
    assert ok, r.stdout[-2000:] + r.stderr[-4000:]


# ------------------------------------------------------------------------------------------------
# b. new data between replays
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_replay_with_new_data(hpc, name):
    case = CASES[name]()
    static = case.make(0)
    a, b = case.run(hpc, static), case.run(hpc, static)
    ok = _same(a, b)
    assert ok, f"{name}: eager is not deterministic, bit equality cannot be the criterion"
    g, out = _capture(lambda: case.run(hpc, static))
    for seed in (1, 2, 3):
        new = case.make(seed)
        for k in case.data:
            static[k].copy_(new[k])
        g.replay()
        got = out.clone()
        ref = case.run(hpc, static)
        torch.cuda.synchronize()
        ok = _same(got, ref)
        assert ok, f"{name}: replay {seed} differs from eager on the same data"


# ------------------------------------------------------------------------------------------------
# c. concurrent replay of graphs captured on the shared default capture stream
# ------------------------------------------------------------------------------------------------
def test_concurrent_replay(hpc):
    """Two FusedMoE graphs and one prefill graph, each GEMM several tile waves deep (about 2000
    tiles over 132 SMs), replayed on two streams without synchronising in between."""
    moe1 = _MoeBlockwise(T=2048, H=2048, I=1024, E=32)
    moe2 = _MoeBlockwise(T=2048, H=2048, I=1024, E=32)
    pre = _Prefill(False, q_total=1800, max_q=1024, kv_cap=2048)
    d1, d2, dp = moe1.make(11), moe2.make(12), pre.make(0)
    ref1, ref2, refp = moe1.run(hpc, d1), moe2.run(hpc, d2), pre.run(hpc, dp)
    ok = _same(ref1, moe1.run(hpc, d1)) and _same(refp, pre.run(hpc, dp))
    assert ok, "eager is not deterministic"
    g1, o1 = _capture(lambda: moe1.run(hpc, d1))
    g2, o2 = _capture(lambda: moe2.run(hpc, d2))
    gp, op = _capture(lambda: pre.run(hpc, dp))
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(torch.cuda.current_stream())
    s2.wait_stream(torch.cuda.current_stream())
    got1, got2, gotp = [], [], []
    for _ in range(5):
        with torch.cuda.stream(s1):
            g1.replay()
            got1.append(o1.clone())
            gp.replay()
            gotp.append(op.clone())
        with torch.cuda.stream(s2):
            g2.replay()
            got2.append(o2.clone())
    torch.cuda.current_stream().wait_stream(s1)
    torch.cuda.current_stream().wait_stream(s2)
    torch.cuda.synchronize()
    bad = [f"{tag} round {r}" for tag, got, ref in (("moe1", got1, ref1), ("moe2", got2, ref2),
                                                    ("prefill", gotp, refp))
           for r, t in enumerate(got) if not _same(t, ref)]
    assert not bad, f"concurrent replays differ from eager: {bad}"
    # eager calls afterwards, on the current stream and on the capture stream itself
    for where, s in (("current stream", torch.cuda.current_stream()),
                     ("capture stream", torch.cuda.graph.default_capture_stream)):
        with torch.cuda.stream(s):
            e1, ep = moe1.run(hpc, d1), pre.run(hpc, dp)
        s.synchronize()
        wrong = [tag for tag, a, b in (("moe", e1, ref1), ("prefill", ep, refp)) if not _same(a, b)]
        assert not wrong, f"eager {wrong} on the {where} after the replays differ from before them"


# ------------------------------------------------------------------------------------------------
# d. many streams
# ------------------------------------------------------------------------------------------------
def _create_streams(n):
    """n new CUDA streams. torch.cuda.Stream() hands out streams from a fixed pool of 32 per
    priority, so distinct handles have to come from cudaStreamCreate itself."""
    cudart = torch.cuda.cudart()
    handles = []
    try:
        for _ in range(n):
            h = ctypes.c_void_p()
            err = cudart.cudaStreamCreate(ctypes.addressof(h))
            assert int(err) == 0, f"cudaStreamCreate failed ({int(err)})"
            handles.append(h.value)
    except BaseException:
        _destroy_streams(handles)
        raise
    return handles


def _destroy_streams(handles):
    torch.cuda.synchronize()
    cudart = torch.cuda.cudart()
    for h in handles:
        cudart.cudaStreamDestroy(h)


def test_many_streams(hpc):
    """200 distinct live streams, each running a blockwise grouped GEMM and a block-sparse prefill,
    all enqueued before any is waited for: every stream needs scheduler counters of its own (the
    eager table must grow past its first chunk, and no two running streams may share a pair), and
    each result must match the one on the default stream."""
    gemm, pre = _GemmBlockwise(), _Prefill(False)
    dg, dp = gemm.make(5), pre.make(0)
    ref_g, ref_p = gemm.run(hpc, dg), pre.run(hpc, dp)
    torch.cuda.synchronize()
    handles = _create_streams(200)
    try:
        streams = [torch.cuda.ExternalStream(h) for h in handles]
        assert len({s.cuda_stream for s in streams}) == 200
        outs = []
        for s in streams:
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                outs.append((gemm.run(hpc, dg), pre.run(hpc, dp)))
        for s in streams:
            torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        bad = [(i, tag) for i, (g, p) in enumerate(outs)
               for tag, t, ref in (("gemm", g, ref_g), ("prefill", p, ref_p)) if not _same(t, ref)]
        del outs
        assert not bad, f"streams {bad[:10]} ({len(bad)} results of 400) were wrong"
    finally:
        _destroy_streams(handles)
