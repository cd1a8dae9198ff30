"""hpc.rope_norm_store_kv and hpc.rope_norm_store_kv_fp8 against the exact fp64 reference
(oracle.rope_exact), on the cases of tests/test_rope_exact_cpu.py: every kernel instantiation,
both V paths, GQA 8/1 to 64/8, head dims 64-320, pages of 16, 24, 32 and 64, split and combined
caches, chunked prefill with zero-row requests, padded decode with mtp 0-3 and positions past 2^16.

Each call is graded element by element: Q, K, V, the FP8 Q scales, the zeroed page tails and every
other byte of a sentinel-filled cache buffer, with no unexplained difference allowed. The bypass
(out_q / out_k / out_v pre-filled with sentinels) must give the cache path's values and leave the
cache untouched. `EXACT <case> ...` lines (visible with -s) give the explained flips per call.
"""
import numpy as np
import pytest
import torch

from oracle import rope_exact as ore
from synth import rope as sr
from test_rope_exact_cpu import CASES, case_id, fp8_args, inputs, misaligned, path_of

pytestmark = pytest.mark.gpu


def _sentinel(shape, fp8):
    if fp8:
        return torch.full(shape, sr.FP8_SENTINEL, dtype=torch.uint8, device="cuda").view(torch.float8_e4m3fn)
    return torch.full(shape, sr.BF16_SENTINEL, dtype=torch.int16, device="cuda").view(torch.bfloat16)


def _call(hpc, c, fp8, bypass):
    """Run one call on the GPU; returns (out dict for ore.grade, cache bits before the call)."""
    inp = inputs(c)
    g = inp["geom"]
    mis = misaligned(c, bypass)
    qkv = inp["qkv"].cuda()
    if "qkv" in mis:
        qkv = sr.at_offset(qkv, 4)
    qw, kw = inp["q_norm_w"].cuda(), inp["k_norm_w"].cuda()
    if "q_norm_w" in mis:
        qw = sr.at_offset(qw, 4)
    if not inp["policy"]:
        qw = kw = None
    flat = _sentinel((g["flat"],), fp8)
    kc, vc = sr.cache_views(flat, g)
    before = ore.bits(flat)
    rows = qkv.shape[0]
    outs = {}
    if bypass:
        outs = dict(out_q=_sentinel((rows, g["hq"], g["dqk"]), fp8),
                    out_k=_sentinel((rows, g["hkv"], g["dqk"]), fp8),
                    out_v=_sentinel((rows, g["hkv"], g["dv"]), fp8))
        if "out_k" in mis:
            outs["out_k"] = sr.at_offset(outs["out_k"], 4)
    args = (kc, vc, qkv, inp["cos_sin"].cuda(), inp["num_seqlen"].cuda(), inp["q_index"].cuda(),
            inp["kv_indices"].cuda(), inp["is_prefill"])
    out = {}
    if fp8:
        fa = fp8_args(c)
        t = lambda x: torch.tensor([x], dtype=torch.float32, device="cuda")  # noqa: E731
        q, qs, flag = hpc.rope_norm_store_kv_fp8(
            *args, t(fa["k_scale"]), t(fa["v_scale"]), fa["quant_policy"],
            max_seqlens=inp["max_seqlens"], upper_max=fa["upper_max"],
            q_scale_inv=t(fa["q_scale_inv"]) if fa["quant_policy"] == 2 else None,
            q_norm_weight=qw, k_norm_weight=kw, qk_norm_policy=inp["policy"], **outs)
        assert int(flag.abs().sum()) == 0 and flag.shape == (inp["num_seqlen"].shape[0], g["hkv"])
        if qs is not None:
            out["q_scale"] = qs.cpu().numpy()
    else:
        q = hpc.rope_norm_store_kv(*args, q_norm_weight=qw, k_norm_weight=kw,
                                   qk_norm_policy=inp["policy"], **outs)
    torch.cuda.synchronize()
    out["q"] = ore.bits(q)
    out["cache"] = ore.bits(flat)
    if bypass:
        assert q.data_ptr() == outs["out_q"].data_ptr()
        out["out_k"] = ore.bits(outs["out_k"])
        out["out_v"] = ore.bits(outs["out_v"]).reshape(rows, -1)
    return out, before


def _slots(inp, cache):
    """K [live rows, Hkv, D] and V [live rows, Hkv * Dv] read back from the cache slots of the rows."""
    g = inp["geom"]
    pos, req = ore.positions(inp["num_seqlen"], inp["q_index"], inp["qkv"].shape[0])
    live = pos >= 0
    p, r = pos[live], req[live]
    cb = inp["kv_indices"].numpy().astype(np.int64)[r, p // g["page"]]
    nk, nv = g["hkv"] * g["dqk"], g["hkv"] * g["dv"]
    k0 = g["k_off"] + cb * g["k_stride"] + (p % g["page"]) * nk
    v0 = g["v_off"] + cb * g["v_stride"] + (p % g["page"]) * nv
    k = cache[k0[:, None] + np.arange(nk)].reshape(len(p), g["hkv"], g["dqk"])
    return k, cache[v0[:, None] + np.arange(nv)], live


def _grade(c, fp8, bypass, out, before, tag):
    inp = inputs(c)
    res = ore.grade(inp, out, fp8, path_of(c, inp, fp8, bypass), fp8_args(c) if fp8 else None, before)
    n = int((ore.positions(inp["num_seqlen"], inp["q_index"], inp["qkv"].shape[0])[0] >= 0).sum())
    flips = {k: v for k, v in res.items() if k.startswith("flips")}
    frac = max(flips.values()) / (n * max(inp["geom"]["hq"], inp["geom"]["hkv"]) * inp["geom"]["dqk"])
    print(f"EXACT {tag} path={path_of(c, inp, fp8, bypass)} {flips} worst_flip_fraction={frac:.2e}")
    assert not ore.failed(res), (tag, res)


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_rope_exact(hpc, c, fp8):
    """The cache path and the bypass, each graded against the fp64 reference; the bypass gives
    the cache path's values (bit for bit when both calls launch the same kernel), writes no cache
    byte, and leaves the rows no request owns untouched."""
    tag = f"{c['name']} {'fp8' if fp8 else 'bf16'}"
    out, before = _call(hpc, c, fp8, False)
    _grade(c, fp8, False, out, before, tag)
    byp, before_b = _call(hpc, c, fp8, True)
    _grade(c, fp8, True, byp, before_b, tag + " bypass")
    inp = inputs(c)
    k, v, live = _slots(inp, out["cache"])
    sent = sr.FP8_SENTINEL if fp8 else sr.BF16_SENTINEL
    for name in ("q", "out_k", "out_v"):
        assert (byp[name][~live] == sent).all(), f"{tag}: bypass wrote {name} of a padding row"
    if path_of(c, inp, fp8, False) == path_of(c, inp, fp8, True):
        assert np.array_equal(byp["q"][live], out["q"][live]), tag
        assert np.array_equal(byp["out_k"][live], k), tag
        assert np.array_equal(byp["out_v"][live], v), tag


def _fp8_raw(num_rows, flag):
    """hpc_rope_norm_store_kv_fp8_async through the C ABI: 3 requests, decode, 8/1 heads."""
    from hpc import _ffi

    hq, hkv, D, page, nreq = 8, 1, 128, 16, 3
    q_lens = [0, 0, 0] if num_rows == 0 else [2, 0, 1]
    dev = "cuda"
    kc = torch.zeros(8, page, hkv, D, dtype=torch.uint8, device=dev)
    vc = torch.zeros_like(kc)
    qkv = torch.randn(num_rows, (hq + 2 * hkv) * D, device=dev).to(torch.bfloat16)
    cos_sin = torch.rand(64, D, device=dev)
    seqlen = torch.tensor([5, 9, 3], dtype=torch.int32, device=dev)
    q_index = torch.tensor([0] + np.cumsum(q_lens).tolist(), dtype=torch.int32, device=dev)
    kv_idx = torch.tensor([[1], [2], [3]], dtype=torch.int32, device=dev)
    out_q = torch.empty(max(num_rows, 1), hq, D, dtype=torch.uint8, device=dev)
    qs = torch.empty(max(num_rows, 1), hq, dtype=torch.float32, device=dev)
    one = torch.ones(1, device=dev)
    p = _ffi.ptr
    rc = _ffi.lib.hpc_rope_norm_store_kv_fp8_async(
        p(out_q), p(kc), p(vc), None, None, p(flag), p(qs), p(qkv) if num_rows else p(out_q),
        p(cos_sin), p(seqlen), p(q_index), p(kv_idx), None, None, p(one), p(one), None, 448.0, 0,
        kc.stride(0), vc.stride(0), nreq, 1, page, num_rows, hq, hkv, D, D, 0, 0, 1,
        _ffi.stream_of(kc))
    _ffi.check(rc, "rope_norm_store_kv_fp8")
    torch.cuda.synchronize()


@pytest.mark.parametrize("num_rows", [0, 3])
def test_rope_fp8_zeroes_split_k_flag(hpc, num_rows):
    """The split-k flags come back zeroed, also from a call with no rows (no kernel runs)."""
    flag = torch.full((3, 1), -7, dtype=torch.int32, device="cuda")
    _fp8_raw(num_rows, flag)
    assert int(flag.abs().sum()) == 0, flag.cpu().tolist()


def test_rope_fp8_then_decode_graph_replay(hpc):
    """rope FP8 -> device-side task map -> FP8 decode captured once; replays on new qkv, lengths
    and page table give what eager calls give on the same data, bit for bit, output and cache."""
    B, hq, hkv, D, page, cap = 8, 32, 8, 128, 64, 1024
    per = cap // page
    npages = B * per + 1
    g0 = torch.Generator().manual_seed(3)
    k8 = (torch.randn(npages, page, hkv, D, generator=g0) * 4).to(torch.float8_e4m3fn).cuda()
    v8 = (torch.randn(npages, page, hkv, D, generator=g0) * 4).to(torch.float8_e4m3fn).cuda()
    k0, v0 = k8.clone(), v8.clone()
    cos_sin = sr.random_cos_sin(cap + 1, D, 4).cuda()
    ks = torch.tensor([0.37], device="cuda")
    vs = torch.tensor([0.21], device="cuda")

    def make(seed):
        g = torch.Generator().manual_seed(seed)
        lens = torch.randint(1, cap + 1, (B,), generator=g, dtype=torch.int32)
        ids = (torch.randperm(npages - 1, generator=g)[:B * per] + 1).int().view(B, per)
        qkv = torch.randn(B, (hq + 2 * hkv) * D, generator=g).to(torch.bfloat16)
        return dict(qkv=qkv.cuda(), lens=lens.cuda(), ids=ids.contiguous().cuda(),
                    q_index=torch.arange(B + 1, dtype=torch.int32, device="cuda"))

    static = make(0)
    tm = hpc.get_attention_decode_task_workspace(B, cap, hkv, 64)

    def run(d):
        q8, qs, _ = hpc.rope_norm_store_kv_fp8(k8, v8, d["qkv"], cos_sin, d["lens"], d["q_index"],
                                               d["ids"], False, ks, vs, 1, max_seqlens=1)
        hpc.assign_attention_decode_task(d["lens"], tm, hkv, 1, True, 64)
        return hpc.attention_decode_fp8(q8, k8, v8, d["ids"], d["lens"], qs, ks, vs, mtp=0,
                                        new_kv_included=True, task_map=tm)

    run(static)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = run(static)
    for seed in (1, 2):
        new = make(seed)
        for key in static:
            static[key].copy_(new[key])
        k8.copy_(k0)
        v8.copy_(v0)
        graph.replay()
        got, gk, gv = out.clone(), k8.clone(), v8.clone()
        k8.copy_(k0)
        v8.copy_(v0)
        ref = run(static)
        torch.cuda.synchronize()
        assert torch.equal(got.view(torch.int16), ref.view(torch.int16)), seed
        assert torch.equal(gk.view(torch.uint8), k8.view(torch.uint8)), seed
        assert torch.equal(gv.view(torch.uint8), v8.view(torch.uint8)), seed
        assert not torch.equal(gk.view(torch.uint8), k0.view(torch.uint8)), seed
