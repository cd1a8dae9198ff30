"""bf16 prefill on the GPU: attention_prefill_bf16 and attention_with_kvcache_prefill_bf16.

a. the reference tests' grids at the reference tolerance (atol 0.016) plus a relative-L2 bound,
   with and without `output=`;
b. the exact check (oracle/prefill_bf16.py) on every case of synth/prefill_bf16.GRID for every input
   family: NHD / HND, pages of 16 / 32 / 64, GQA groups 1 / 4 / 8, ragged and chunked requests,
   sq = 0 slots, an oversized max_seqlens_q;
c. the dense and paged ops agree bit for bit on the same data, and repeated calls are bit-identical;
d. a cache written by rope_norm_store_kv (prefill, 16-token pages) is read correctly;
e. CUDA-graph capture: replay on new data equals eager, and replays on two streams next to a captured
   FP8 prefill.
"""
import math

import pytest
import torch

from oracle import prefill_bf16 as ob
from synth import prefill_bf16 as sb

pytestmark = pytest.mark.gpu

REL_L2 = 0.01


def _run(hpc, d, output=None):
    if d["op"] == "dense":
        return hpc.attention_prefill_bf16(d["q"], d["k"], d["v"], d["seqlens_q"], d["cu_seqlens_q"],
                                          d["max_q"], output=output)
    return hpc.attention_with_kvcache_prefill_bf16(d["q"], d["kcache"], d["vcache"], d["cu_seqlens_q"],
                                                   d["block_ids"], d["seqlens_kv"], d["max_q"],
                                                   output=output)


def _reference_check(out, gt):
    out, gt = out.float(), gt.float()
    err = (out - gt).abs()
    assert float(err.max()) <= 0.016, f"max |err| {float(err.max()):.4f}"
    rel = float((out - gt).norm() / gt.norm())
    assert rel <= REL_L2, f"rel L2 {rel:.4g}"


def _cpu(d):
    return {k: (v.cpu() if isinstance(v, torch.Tensor) else v) for k, v in d.items()}


# ------------------------------------------------------------------------------------------------
# a. reference grids
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("use_output", [True, False])
@pytest.mark.parametrize("seq", [2007, 3907])
@pytest.mark.parametrize("num_batch", [1, 4])
def test_prefill_reference_grid(hpc, num_batch, seq, use_output):
    d = sb.make_reference_case("dense", [seq] * num_batch, hq=4, hkv=1, seed=seq + num_batch,
                               device="cuda")
    out = torch.empty_like(d["q"]) if use_output else None
    y = _run(hpc, d, out)
    if use_output:
        assert y.data_ptr() == out.data_ptr()
    gt = ob.varlen_prefill(d["q"], d["k"], d["v"], d["cu_seqlens_q"].cpu())
    _reference_check(y, gt)


@pytest.mark.parametrize("use_output", [True, False])
@pytest.mark.parametrize("seq_kv", [1500, 3000])
@pytest.mark.parametrize("seq_q", [100, 500, 1000, 1500])
@pytest.mark.parametrize("num_batch", [1, 2, 4, 8])
def test_kvcache_prefill_reference_grid(hpc, num_batch, seq_q, seq_kv, use_output):
    d = sb.make_reference_case("paged", [seq_q] * num_batch, [seq_kv] * num_batch, hq=4, hkv=1,
                               page=64, seed=seq_q * 7 + seq_kv + num_batch, device="cuda")
    out = torch.empty_like(d["q"]) if use_output else None
    y = _run(hpc, d, out)
    if use_output:
        assert y.data_ptr() == out.data_ptr()
    gt = ob.kvcache_prefill(d["q"], d["kcache"], d["vcache"], d["cu_seqlens_q"].cpu(),
                            d["block_ids"].cpu(), d["seqlens_kv"].cpu())
    _reference_check(y, gt)


# ------------------------------------------------------------------------------------------------
# b. exact check
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", sb.KINDS)
@pytest.mark.parametrize("case", sb.GRID, ids=sb.case_id)
def test_exact(hpc, case, kind):
    d = sb.make_exact_case(case, kind, device="cuda")
    y = _run(hpc, d)
    torch.cuda.synchronize()
    r = ob.check(y.cpu(), _cpu(d))
    assert r["nan_ok"], "NaN rows differ from the exact reference"
    assert r["ok_a"], f"|out - exact| / B = {r['worst']:.3f} > 1"
    assert r["ok_b"], f"rel L2 {r['rel']:.4g} vs lossy oracle {r['rel_oracle']:.4g}"


def test_every_row_written(hpc):
    """Every row of every request is written, next to a request with no new token (which owns no
    row) and with an oversized max_seqlens_q."""
    case = sb.GRID[3]  # has an sq = 0 slot between two requests
    d = sb.make_exact_case(case, "peaked", device="cuda")
    out = torch.full_like(d["q"], math.nan)
    _run(hpc, d, out)
    assert not bool(torch.isnan(out).any())


# ------------------------------------------------------------------------------------------------
# c. dense == paged, determinism
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("page", [16, 32, 64])
def test_dense_equals_paged(hpc, page):
    q_lens = [1, 300, 0, 517, 128]
    d = sb.make_reference_case("dense", q_lens, hq=8, hkv=2, seed=page, device="cuda")
    gen = torch.Generator().manual_seed(page)
    nblk = [(n + page - 1) // page for n in q_lens]
    num_blocks = sum(nblk) + 2
    perm = torch.randperm(num_blocks, generator=gen).to(torch.int32)
    ids = torch.zeros(len(q_lens), max(nblk), dtype=torch.int32)
    kc = torch.zeros(num_blocks, page, 2, 128, dtype=torch.bfloat16, device="cuda")
    vc = torch.zeros_like(kc)
    cu, s0 = 0, 0
    for b, n in enumerate(q_lens):
        ids[b, :nblk[b]] = perm[cu:cu + nblk[b]]
        cu += nblk[b]
        for j in range(nblk[b]):
            rows = slice(s0 + j * page, min(s0 + (j + 1) * page, s0 + n))
            m = rows.stop - rows.start
            kc[int(ids[b, j]), :m] = d["k"][rows]
            vc[int(ids[b, j]), :m] = d["v"][rows]
        s0 += n
    p = dict(op="paged", q=d["q"], kcache=kc, vcache=vc, cu_seqlens_q=d["cu_seqlens_q"],
             block_ids=ids.cuda(), seqlens_kv=d["seqlens_q"], max_q=d["max_q"])
    yd, yp = _run(hpc, d), _run(hpc, p)
    assert torch.equal(yd, yp)
    for _ in range(3):
        assert torch.equal(_run(hpc, d), yd) and torch.equal(_run(hpc, p), yp)


# ------------------------------------------------------------------------------------------------
# d. cache written by rope_norm_store_kv
# ------------------------------------------------------------------------------------------------
def test_cache_from_rope_norm_store_kv(hpc):
    from synth import rope as sr

    r = sr.make_inputs(5, True, None, 16, 2, 128, kv_block_size=16, max_num_kv_blocks=160,
                       max_rope_position=2048, seed=3, len_range=(100, 400))
    c = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in r.items()}
    q = hpc.rope_norm_store_kv(c["kcache"], c["vcache"], c["qkv"], c["cos_sin"], c["num_seqlen"],
                               c["q_index"], c["kv_indices"], True, c["q_norm_w"], c["k_norm_w"],
                               qk_norm_policy=2)
    q_lens = (r["q_index"][1:] - r["q_index"][:-1]).tolist()
    d = dict(op="paged", q=q, kcache=c["kcache"], vcache=c["vcache"], cu_seqlens_q=c["q_index"],
             block_ids=c["kv_indices"], seqlens_kv=c["num_seqlen"], max_q=max(q_lens))
    y = _run(hpc, d)
    torch.cuda.synchronize()
    ob_out = ob.check(y.cpu(), _cpu(d))
    assert ob_out["ok_a"] and ob_out["ok_b"], ob_out


# ------------------------------------------------------------------------------------------------
# e. CUDA graphs
# ------------------------------------------------------------------------------------------------
def _capture(fn):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn()
    return g, out


def _fill(static, new):
    for k, v in new.items():
        if isinstance(v, torch.Tensor):
            static[k].copy_(v)


def test_graph_replay_new_data(hpc):
    for case in (sb.GRID[0], sb.GRID[4]):
        static = sb.make_exact_case(case, "peaked", device="cuda")
        g, out = _capture(lambda: _run(hpc, static))
        for kind in sb.KINDS:
            _fill(static, sb.make_exact_case(case, kind, device="cuda"))
            g.replay()
            torch.cuda.synchronize()
            got = out.clone()
            ref = _run(hpc, static)
            torch.cuda.synchronize()
            assert torch.equal(got, ref), f"{sb.case_id(case)} {kind}: replay differs from eager"


def test_graph_concurrent_with_fp8_prefill(hpc):
    from synth.prefill import make_inputs

    dd = sb.make_exact_case(sb.GRID[2], "needle", device="cuda")
    dp = sb.make_exact_case(sb.GRID[4], "needle", device="cuda")
    f8 = make_inputs([900, 700], [1500, 1200], 8, 2, 0.3, False, seed=5, device="cuda")
    f8["block_mask"] = f8["block_mask"].to(torch.uint8).contiguous()

    def fp8():
        return hpc.attention_with_kvcache_blocksparse_prefill_fp8(
            f8["q"], f8["kcache"], f8["vcache"], f8["qscale"], f8["kscale"], f8["vscale"],
            f8["cu_seqlens_q"], f8["block_ids"], f8["seqlens_kv"], f8["max_q"],
            block_mask=f8["block_mask"])

    fns = (lambda: _run(hpc, dd), lambda: _run(hpc, dp), fp8)
    refs = [f() for f in fns]
    torch.cuda.synchronize()
    graphs = [_capture(f) for f in fns]
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(torch.cuda.current_stream())
    s2.wait_stream(torch.cuda.current_stream())
    got = [[], [], []]
    for _ in range(4):
        with torch.cuda.stream(s1):
            graphs[0][0].replay()
            got[0].append(graphs[0][1].clone())
            graphs[2][0].replay()
            got[2].append(graphs[2][1].clone())
        with torch.cuda.stream(s2):
            graphs[1][0].replay()
            got[1].append(graphs[1][1].clone())
    torch.cuda.current_stream().wait_stream(s1)
    torch.cuda.current_stream().wait_stream(s2)
    torch.cuda.synchronize()
    bad = [f"{i} round {r}" for i in range(3) for r, t in enumerate(got[i])
           if not torch.equal(t.view(torch.int16), refs[i].view(torch.int16))]
    assert not bad, f"concurrent replays differ from eager: {bad}"
