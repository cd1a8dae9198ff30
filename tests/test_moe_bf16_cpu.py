"""CPU checks of the bf16 FusedMoE's oracle, inputs and argument checks (no GPU needed).

The oracle's stage checks are run on a kernel emulated from the contract in fp32 torch
(oracle.moe_bf16.reference_fp32 and its stages): they must pass it, and must catch planted bugs."""
import ctypes
import importlib

import pytest
import torch

from oracle import moe_bf16 as ob, moe_exact as ox
from synth.moe_bf16 import make_group_gemm_bf16_inputs, make_moe_bf16_inputs


def _emulate(d):
    """Every scratch tensor of the bf16 pipeline from an fp32 torch restatement of each stage, and
    the output."""
    E = d["gate_up_weight"].size(0)
    r = ob.route(d["topk_ids"], E, d["rank_ep"], d["num_expert_total"])
    gathered = d["x"][r["src_token"]]
    inter = d["gate_up_weight"].size(1) // 2
    rows = gathered.size(0)
    down_input = torch.empty((rows, inter), dtype=torch.bfloat16)
    down_output = torch.empty((rows, d["x"].size(1)), dtype=torch.bfloat16)
    for e in range(E):
        sl = slice(int(r["cu"][e]), int(r["cu"][e + 1]))
        gu = (gathered[sl].float() @ d["gate_up_weight"][e].float().t()).to(torch.bfloat16)
        down_input[sl] = ob.silu_mul(gu[:, :inter], gu[:, inter:]).to(torch.bfloat16)
        down_output[sl] = (down_input[sl].float() @ d["down_weight"][e].float().t()).to(torch.bfloat16)
    pos = r["topk_pos"].long()
    terms = down_output.float()[pos.clamp_min(0)] * (pos >= 0)[..., None] * d["topk_scale"][..., None]
    y = torch.zeros(d["x"].shape)
    for k in range(pos.size(1)):
        y += terms[:, k]
    if d["shared_output"] is not None:
        y += d["shared_output"].float()
    tiles = (r["counts"] + 127) // 128
    cu_tiles = torch.zeros(E + 1, dtype=torch.int32)
    cu_tiles[1:] = torch.cumsum(tiles, 0)
    s = dict(counts=r["counts"], cu_counts=r["cu"], topk_pos=r["topk_pos"], gate_up_input=gathered,
             tiles=tiles.to(torch.int32), cu_tiles=cu_tiles, down_input=down_input,
             down_output=down_output)
    return r, s, y.to(torch.bfloat16)


def _check(d, r, s, y):
    ob.check_route(r, d["x"], s)
    rows = ob.rows_to_check(r)
    ob.check_gateup(s["gate_up_input"], r, d["gate_up_weight"], rows, s["down_input"])
    yd, B = ob.down_exact(s["down_input"], r, d["down_weight"], rows)
    ox.check_down(s["down_output"][rows], yd, B)
    ox.accumulation_probe(s["down_output"][rows], yd, B)
    o, B = ox.reduce_exact(s["down_output"], s["topk_pos"], d["topk_scale"], d["shared_output"])
    ox.check_down(y, o, B, tag="reduce")
    ox.accumulation_probe(y, o, B, tag="reduce")


CASES = [dict(T=37, k=2, H=256, I=128, E=8),
         dict(T=5, k=4, H=384, I=256, E=16, routing="sparse"),
         dict(T=60, k=2, H=256, I=128, E=16, routing="other_rank", size_ep=4, rank_ep=3, shared=True),
         dict(T=50, k=2, H=256, I=128, E=8, routing="hot")]


def _make(c, seed=5):
    return make_moe_bf16_inputs(c["T"], c["k"], c["H"], c["I"], c["E"], routing=c.get("routing", "uniform"),
                                size_ep=c.get("size_ep", 1), rank_ep=c.get("rank_ep", 0),
                                shared=c.get("shared", False), seed=seed)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_oracle_passes_fp32_restatement(case):
    d = _make(CASES[case])
    r, s, y = _emulate(d)
    _check(d, r, s, y)
    # the naive per-token restatement agrees with the staged emulation up to fp32 summation order
    # (a batched and a one-row matmul add in different orders)
    naive = ob.reference_fp32(d["x"], d["gate_up_weight"], d["down_weight"], d["topk_ids"],
                              d["topk_scale"], d["rank_ep"], d["num_expert_total"], d["shared_output"])
    torch.testing.assert_close(naive.float(), y.float(), atol=2e-2, rtol=2e-2)


def test_gateup_emulation_matches_restatement():
    d = _make(CASES[0])
    r, s, _ = _emulate(d)
    rows = ob.rows_to_check(r)
    em = ob.gateup_emulate(s["gate_up_input"], r, d["gate_up_weight"], rows)
    d_ = (ob.bf16_ordinal(em) - ob.bf16_ordinal(s["down_input"][rows])).abs()
    assert int(d_.max()) <= 1 and float((d_ > 0).float().mean()) < 1e-3


@pytest.mark.parametrize("bug", ["swap_gate_up", "no_gate_round", "row_order", "down_scale",
                                 "reduce_skip", "tiles"])
def test_bug_caught(bug):
    d = _make(CASES[0])
    r, s, y = _emulate(d)
    inter = d["gate_up_weight"].size(1) // 2
    if bug == "swap_gate_up":
        gu = torch.cat([d["gate_up_weight"][:, inter:], d["gate_up_weight"][:, :inter]], 1)
        r2, s2, y2 = _emulate(dict(d, gate_up_weight=gu))
        s["down_input"] = s2["down_input"]
    elif bug == "no_gate_round":
        e = int(r["expert_of_row"][0])
        gu = s["gate_up_input"][:1].float() @ d["gate_up_weight"][e].float().t()
        s["down_input"][0] = ob.silu_mul(gu[:, :inter], gu[:, inter:].to(torch.bfloat16)).to(torch.bfloat16)[0]
        s["down_input"][0] = s["down_input"][0] * 1.02
    elif bug == "row_order":
        s["gate_up_input"] = s["gate_up_input"].flip(0)
    elif bug == "down_scale":
        s["down_output"] = (s["down_output"].float() * 1.01).to(torch.bfloat16)
    elif bug == "reduce_skip":
        y = (y.float() - s["down_output"].float()[r["topk_pos"][:, 1].long()]
             * d["topk_scale"][:, 1:2]).to(torch.bfloat16)
    elif bug == "tiles":
        s["tiles"] = r["counts"] // 64
    with pytest.raises(AssertionError):
        _check(d, r, s, y)


def test_synth_deterministic():
    for c in CASES:
        a, b = _make(c, seed=9), _make(c, seed=9)
        for k, v in a.items():
            if isinstance(v, torch.Tensor):
                assert torch.equal(v, b[k]), k
            else:
                assert v == b[k], k
        other = _make(c, seed=10)
        assert not torch.equal(a["x"], other["x"])
    g1 = make_group_gemm_bf16_inputs([3, 0, 5], 128, 128)
    g2 = make_group_gemm_bf16_inputs([3, 0, 5], 128, 128)
    assert all(torch.equal(g1[k], g2[k]) for k in g1)
    assert g1["cu_seqlens"].tolist() == [0, 3, 3, 8]


def test_group_gemm_oracle():
    d = make_group_gemm_bf16_inputs([0, 7, 0, 20], 256, 128)
    want, B = ob.group_gemm_exact(d["x"], d["weight"], d["seqlens"], d["cu_seqlens"])
    y = torch.full_like(want, float("nan")).to(torch.bfloat16)
    for g in range(4):
        n, r0 = int(d["seqlens"][g]), int(d["cu_seqlens"][g])
        y[r0:r0 + n] = (d["x"][r0:r0 + n].float() @ d["weight"][g].float().t()).to(torch.bfloat16)
    inside = ~torch.isnan(want[:, 0])
    assert int(inside.sum()) == 27
    ox.check_down(y[inside], want[inside], B[inside])
    with pytest.raises(AssertionError):
        ox.check_down((y[inside].float() * 1.01).to(torch.bfloat16), want[inside], B[inside])


# ---- argument checks: every limit raises with its message before any device work ---------------
def _bf16_args(T=4, H=256, I=128, E=8, k=2):
    return dict(x=torch.zeros(T, H, dtype=torch.bfloat16),
                gate_up_weight=torch.zeros(E, 2 * I, H, dtype=torch.bfloat16),
                down_weight=torch.zeros(E, H, I, dtype=torch.bfloat16),
                topk_ids=torch.zeros(T, k, dtype=torch.int32), topk_scale=torch.zeros(T, k),
                rank_ep=0, num_expert_total=E, shared_output=None, output=None)


def test_wrapper_rejects_bad_input(hpc):
    fm = importlib.import_module("hpc.fuse_moe")

    def bad(match, **kw):
        a = {**_bf16_args(), **kw}
        with pytest.raises(RuntimeError, match=match):
            fm._fuse_moe_bf16_impl(**a)

    a = _bf16_args()
    bad("x must be torch.bfloat16", x=a["x"].float())
    bad("gate_up_weight must be torch.bfloat16", gate_up_weight=a["gate_up_weight"].half())
    bad("topk_ids must be torch.int32", topk_ids=a["topk_ids"].long())
    bad("topk_scale must be torch.float32", topk_scale=a["topk_scale"].double())
    bad("x must be contiguous", x=torch.zeros(256, 4, dtype=torch.bfloat16).t())
    bad("hidden 192 must be a positive multiple of 128", **_bf16_args(H=192))
    bad("gate_up_weight rows 192", gate_up_weight=torch.zeros(8, 192, 256, dtype=torch.bfloat16))
    bad("intermediate|rows 160", **{**_bf16_args(I=80)})
    bad("down_weight must be", down_weight=torch.zeros(8, 256, 256, dtype=torch.bfloat16))
    bad("gate_up_weight hidden 384", gate_up_weight=torch.zeros(8, 256, 384, dtype=torch.bfloat16))
    bad("local experts 513", **_bf16_args(E=513))
    bad("num_expert_total 4 below", num_expert_total=4)
    bad("num_topk 129", **_bf16_args(k=129))
    bad("topk_ids and topk_scale", topk_scale=torch.zeros(4, 3))
    bad("shared_output must be", shared_output=torch.zeros(4, 128, dtype=torch.bfloat16))
    bad("output must be", output=torch.zeros(4, 256))
    bad("CUDA tensor")

    gg = importlib.import_module("hpc.group_gemm")
    x = torch.zeros(10, 256, dtype=torch.bfloat16)
    w = torch.zeros(3, 128, 256, dtype=torch.bfloat16)
    sl, cu = torch.zeros(3, dtype=torch.int32), torch.zeros(4, dtype=torch.int32)

    def bad_gg(match, **kw):
        a = {**dict(x=x, weight=w, seqlens=sl, cu_seqlens=cu, output=None), **kw}
        with pytest.raises(RuntimeError, match=match):
            gg._group_gemm_bf16_impl(**a)

    bad_gg("K 192", x=torch.zeros(10, 192, dtype=torch.bfloat16),
           weight=torch.zeros(3, 128, 192, dtype=torch.bfloat16))
    bad_gg("N 64", weight=torch.zeros(3, 64, 256, dtype=torch.bfloat16))
    bad_gg("weight K 128 differs", weight=torch.zeros(3, 128, 128, dtype=torch.bfloat16))
    bad_gg("groups 513", weight=torch.zeros(513, 128, 256, dtype=torch.bfloat16),
           seqlens=torch.zeros(513, dtype=torch.int32), cu_seqlens=torch.zeros(514, dtype=torch.int32))
    bad_gg("seqlens must be", seqlens=torch.zeros(2, dtype=torch.int32))
    bad_gg("x must be torch.bfloat16", x=x.float())
    bad_gg("CUDA tensor")


def _buf(n, align_off=0):
    b = ctypes.create_string_buffer(n + 64)
    return b, ((ctypes.addressof(b) + 15) // 16) * 16 + align_off


def test_launchers_reject_bad_arguments(hpc):
    lib = hpc._ffi.lib
    _keep, p = _buf(1 << 12)

    def call(T=4, H=256, I=128, k=2, Et=8, E=8, rank=0, x=p):
        return lib.hpc_fuse_moe_bf16_async(p, x, p, p, p, p, p, p, p, p, p, p, p, p, None, T, H, I,
                                           k, Et, E, rank, None)

    for kw, msg in ((dict(T=-1), b"negative"), (dict(E=0), b"local experts 0"),
                    (dict(E=513, Et=513), b"local experts 513"), (dict(Et=4), b"below"),
                    (dict(k=0), b"num_topk 0"), (dict(k=129), b"num_topk 129"),
                    (dict(H=192), b"hidden (192)"), (dict(I=64), b"intermediate (64)"),
                    (dict(x=p + 4), b"16-byte aligned")):
        assert call(**kw) == 1, kw
        assert msg in lib.hpc_last_error(), (kw, lib.hpc_last_error())
    assert call(T=0) == 0  # no launch

    def gg(G=3, m=10, n=128, k=256, x=p):
        return lib.hpc_group_gemm_bf16_async(p, x, p, p, p, G, m, n, k, None)

    for kw, msg in ((dict(G=0), b"num_group 0"), (dict(G=513), b"num_group 513"),
                    (dict(k=192), b"k (192)"), (dict(n=64), b"n (64)"), (dict(m=-1), b"negative"),
                    (dict(x=p + 8), b"16-byte aligned")):
        assert gg(**kw) == 1, kw
        assert msg in lib.hpc_last_error(), (kw, lib.hpc_last_error())
    assert gg(m=0) == 0


def test_exports_and_fake_shapes(hpc):
    from torch._subclasses.fake_tensor import FakeTensorMode

    assert hpc.fuse_moe_bf16 is importlib.import_module("hpc.fuse_moe").fuse_moe_bf16
    assert hpc.group_gemm_bf16 is importlib.import_module("hpc.group_gemm").group_gemm_bf16
    with FakeTensorMode():
        a = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in _bf16_args().items()}
        y = torch.ops.hpc.fuse_moe_bf16(a["x"], a["gate_up_weight"], a["down_weight"], a["topk_ids"],
                                        a["topk_scale"], 0, 8, None, None)
        assert y.shape == (4, 256) and y.dtype == torch.bfloat16
        x = torch.empty(10, 256, dtype=torch.bfloat16, device="cuda")
        w = torch.empty(3, 384, 256, dtype=torch.bfloat16, device="cuda")
        sl = torch.empty(3, dtype=torch.int32, device="cuda")
        y = torch.ops.hpc.group_gemm_bf16(x, w, sl, torch.empty(4, dtype=torch.int32, device="cuda"),
                                          None)
        assert y.shape == (10, 384) and y.dtype == torch.bfloat16
