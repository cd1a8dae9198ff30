"""Absorbed MLA decode (hpc.attention_decode_mla_bf16, csrc/decode_attn_mla.cu) against the exact
fp64 reference of oracle/attention_mla.py: element-wise bound and aggregate check, every head
count and MTP depth, page and tile edges, split-k schedules from both schedulers and from inside
the call, NaN in every unused cache slot, strided cache and output, repeatability and CUDA-graph
replay."""
import math

import pytest
import torch

from oracle import attention_mla as om
from synth import attention_mla as sm

pytestmark = pytest.mark.gpu

HEADS = (8, 16, 32, 64, 128)
MTPS = (0, 1, 3)


def _ctas(hpc):
    return hpc._ffi.sm_count(torch.device("cuda", 0))


def _run(hpc, d, map_from="gpu", new_kv_included=True, kv=None, output=None):
    dev = "cuda"
    q = d["q"].to(dev)
    kv = d["kv"].to(dev) if kv is None else kv
    ids = d["block_ids"].to(dev)
    sq = d["num_seq_q"]
    lens = d["lens_total"] if new_kv_included else d["lens_total"] - sq
    T = om.num_tiles(d["h"], sq)
    tm = None
    if map_from != "none":
        tm = hpc.get_attention_decode_task_workspace(len(lens), int(ids.size(1)) * 64 + sq, T,
                                                     d["min_process_len"], device=dev)
        src = lens.to(dev) if map_from == "gpu" else lens
        hpc.assign_attention_decode_task(src, tm, T, sq, new_kv_included, d["min_process_len"])
    y = hpc.attention_decode_mla_bf16(q, kv, ids, lens.to(dev), d["scale"], mtp=d["mtp"],
                                      new_kv_included=new_kv_included, task_map=tm, output=output)
    torch.cuda.synchronize()
    return y


def _check(y, d, tag):
    r = om.check(y.float().cpu(), d, tag)
    print(f"EXACT mla {tag} worst={r['worst']:.3f} rel={r['rel']:.3g} oracle_rel={r['rel_oracle']:.3g}")
    assert r["nan_ok"] and r["ok_a"] and r["ok_b"], (tag, r)
    return r


@pytest.mark.parametrize("h", HEADS)
@pytest.mark.parametrize("mtp", MTPS)
def test_mla_exact_heads_mtp(hpc, h, mtp):
    sq = mtp + 1
    for i, kind in enumerate(sm.KINDS):
        d = sm.make_case(sm.lengths(sq), h, mtp, seed=100 * h + 10 * mtp + i, kind=kind,
                         num_total_ctas=_ctas(hpc), min_process_len=64)
        _check(_run(hpc, d), d, f"h{h} mtp{mtp} {kind}")


@pytest.mark.parametrize("map_from", ["gpu", "cpu", "none"])
@pytest.mark.parametrize("new_kv_included", [True, False])
def test_mla_task_map_sources(hpc, map_from, new_kv_included):
    mpl = 512 if map_from == "none" else 64
    d = sm.make_case([3000, 65, 2, 700, 129], 128, 1, seed=7, scale=sm.SCALE_PLAIN,
                     num_total_ctas=_ctas(hpc), min_process_len=mpl)
    _check(_run(hpc, d, map_from, new_kv_included), d, f"map {map_from} nkv {new_kv_included}")


@pytest.mark.parametrize("h", [16, 128])
def test_mla_long_request_every_cta(hpc, h):
    d = sm.make_case([40000], h, 0, seed=11, num_total_ctas=_ctas(hpc), min_process_len=64)
    # 313 tiles of 128 keys per query tile, cut into chunks of P = ceil(313 T / SMs) tiles
    T = om.num_tiles(h, 1)
    P = -(-313 * T // _ctas(hpc))
    assert len(d["chunks"][(0, 0)]) == -(-313 // P) > 50
    _check(_run(hpc, d), d, f"long h{h}")


def test_mla_many_short_requests(hpc):
    g = torch.Generator().manual_seed(5)
    lens = (torch.randint(2, 300, (300,), generator=g)).tolist()
    d = sm.make_case(lens, 16, 1, seed=6, num_total_ctas=_ctas(hpc), min_process_len=64)
    _check(_run(hpc, d), d, "many short")


def test_mla_strided_cache_and_output(hpc):
    d = sm.make_case([500, 64, 1300], 32, 1, seed=9, num_total_ctas=_ctas(hpc), min_process_len=64)
    wide = torch.full((d["kv"].size(0), 64, 640), math.nan, dtype=torch.bfloat16, device="cuda")
    wide[..., :576] = d["kv"].cuda()
    kv = wide[..., :576]
    assert kv.stride(1) == 640
    rows = d["q"].size(0)
    buf = torch.full((rows, 32 * 512 + 64), math.nan, dtype=torch.bfloat16, device="cuda")
    out = buf[:, :32 * 512].view(rows, 32, 512)
    y = _run(hpc, d, kv=kv, output=out)
    assert y.data_ptr() == out.data_ptr()
    assert torch.isnan(buf[:, 32 * 512:]).all()
    _check(y, d, "strided")


def test_mla_repeatable_bits(hpc):
    d = sm.make_case([5000, 300, 77], 128, 0, seed=3, num_total_ctas=_ctas(hpc), min_process_len=64)
    a = _run(hpc, d)
    b = _run(hpc, d)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_mla_graph_capture_replay(hpc):
    ctas = _ctas(hpc)
    d1 = sm.make_case([900, 70, 2000], 64, 1, seed=21, num_total_ctas=ctas, min_process_len=64)
    d2 = sm.make_case([1500, 300, 10], 64, 1, seed=22, num_total_ctas=ctas, min_process_len=64)
    nblk = max(d1["kv"].size(0), d2["kv"].size(0))
    mb = max(d1["block_ids"].size(1), d2["block_ids"].size(1))
    kv = torch.zeros(nblk, 64, 576, dtype=torch.bfloat16, device="cuda")
    ids = torch.zeros(3, mb, dtype=torch.int32, device="cuda")
    q = torch.zeros_like(d1["q"], device="cuda")
    lens = torch.zeros(3, dtype=torch.int32, device="cuda")
    T = om.num_tiles(64, 2)
    tm = hpc.get_attention_decode_task_workspace(3, mb * 64 + 2, T, 64, device="cuda")

    def load(d):
        kv.zero_()
        kv[:d["kv"].size(0)] = d["kv"].cuda()
        ids.zero_()
        ids[:, :d["block_ids"].size(1)] = d["block_ids"].cuda()
        q.copy_(d["q"].cuda())
        lens.copy_(d["lens_total"].cuda())

    load(d1)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        hpc.assign_attention_decode_task(lens, tm, T, 2, True, 64)
        hpc.attention_decode_mla_bf16(q, kv, ids, lens, d1["scale"], mtp=1, new_kv_included=True,
                                      task_map=tm)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        hpc.assign_attention_decode_task(lens, tm, T, 2, True, 64)
        y = hpc.attention_decode_mla_bf16(q, kv, ids, lens, d1["scale"], mtp=1,
                                          new_kv_included=True, task_map=tm)
    for d, tag in ((d1, "graph 1"), (d2, "graph 2")):
        load(d)
        g.replay()
        torch.cuda.synchronize()
        _check(y, d, tag)


def test_mla_rejections(hpc):
    dev = "cuda"
    q = torch.zeros(2, 16, 576, dtype=torch.bfloat16, device=dev)
    kv = torch.zeros(4, 64, 576, dtype=torch.bfloat16, device=dev)
    ids = torch.zeros(2, 2, dtype=torch.int32, device=dev)
    lens = torch.full((2,), 10, dtype=torch.int32, device=dev)
    f = hpc.attention_decode_mla_bf16
    f(q, kv, ids, lens, 0.1)
    bad = [
        lambda: f(torch.zeros(2, 12, 576, dtype=torch.bfloat16, device=dev), kv, ids, lens, 0.1),
        lambda: f(torch.zeros(2, 256, 576, dtype=torch.bfloat16, device=dev), kv, ids, lens, 0.1),
        lambda: f(q, kv, ids, lens, 0.1, mtp=4),
        lambda: f(q, kv, ids, lens, 0.1, mtp=1),
        lambda: f(q.float(), kv, ids, lens, 0.1),
        lambda: f(q, kv.half(), ids, lens, 0.1),
        lambda: f(q, torch.zeros(4, 32, 576, dtype=torch.bfloat16, device=dev), ids, lens, 0.1),
        lambda: f(q, torch.zeros(4, 64, 640, dtype=torch.bfloat16, device=dev)[..., 1:577], ids,
                  lens, 0.1),
        lambda: f(q, torch.zeros(4, 64, 580, dtype=torch.bfloat16, device=dev)[..., :576], ids,
                  lens, 0.1),
        lambda: f(q[:, :, :512], kv, ids, lens, 0.1),
        lambda: f(q, kv, ids.long(), lens, 0.1),
        lambda: f(q, kv, ids, lens, 0.1, output=torch.zeros(2, 16, 128, dtype=torch.bfloat16,
                                                             device=dev)),
        lambda: f(torch.zeros(2049, 8, 576, dtype=torch.bfloat16, device=dev), kv,
                  torch.zeros(2049, 2, dtype=torch.int32, device=dev),
                  torch.full((2049,), 10, dtype=torch.int32, device=dev), 0.1),
    ]
    for i, call in enumerate(bad):
        with pytest.raises(RuntimeError):
            call()
            torch.cuda.synchronize()
            raise AssertionError(f"case {i} was accepted")
