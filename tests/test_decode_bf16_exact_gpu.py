"""bf16 paged decode (hpc.attention_decode_bf16) against the exact fp64 reference
(oracle.prefill_bf16.decode_exact), on inputs built so that every key, page, MTP row and split-k
chunk shows in the output (synth.attention_exact.make_decode_bf16_exact_inputs).

Each run passes (a) |kernel - exact| <= B element-wise and (b) rel L2 of the kernel's error
<= AGG_C times the lossy oracle's + AGG_FLOOR, and prints one line `EXACT <tag> worst=...
rel=... rel_oracle=...` (visible with -s). The bound and the mutation-checked case list are
shared with tests/test_decode_bf16_exact_cpu.py; here the split-k chunks come from the schedule
of this device's CTA count.
"""
import pytest
import torch

from oracle import attention_exact as ox
from synth import rope as sr
from test_decode_bf16_exact_cpu import (CASES, PAGES, build, case_id, chunks_of, coverage, exact,
                                        lossy)
from synth.attention_exact import make_decode_bf16_exact_inputs

pytestmark = pytest.mark.gpu


def _ctas():
    from hpc import attention as ha

    return ha._num_total_ctas()


def _run(hpc, d, sq, hkv, mpl, task_map="gpu", new_kv_included=True):
    lens = d["kv_lens_total"]
    arg = lens if new_kv_included else lens - sq
    tm = None
    if task_map is not None:
        tm = hpc.get_attention_decode_task_workspace(lens.numel(), int(lens.max()), hkv, mpl)
        hpc.assign_attention_decode_task(arg.cpu() if task_map == "cpu" else arg, tm, hkv, sq,
                                         new_kv_included, mpl)
    kv = d["kvcache"]
    return hpc.attention_decode_bf16(d["q"], kv[:, 0], kv[:, 1], d["block_ids"], arg, mtp=sq - 1,
                                     new_kv_included=new_kv_included, splitk=True,
                                     task_map=tm).cpu()


def _report(tag, out, d, sq, chunks):
    y, bound = exact(d, sq, chunks)
    r = ox.assert_exact(out, y, bound, lossy(d, sq, chunks), tag)
    print(f"EXACT {tag} worst={r['worst']:.4f} rel={r['rel']:.3e} rel_oracle={r['rel_oracle']:.3e}")


@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_decode_bf16_exact_cases(hpc, c):
    d, ch = build(c, _ctas(), device="cuda")
    cov = coverage(d, ch, c["page"])
    assert cov["single"] and cov["multi"], cov
    if c["kind"] == "needle":
        assert cov["needle_past_first"], cov
    _report(f"decode bf16 {case_id(c)}", _run(hpc, d, c["sq"], c["hkv"], c["mpl"]), d, c["sq"], ch)


def test_decode_bf16_exact_cases_reach_long_chunks():
    """On this device's schedule too, each page size has a chunk longer than 32 pages."""
    for page in PAGES:
        assert any(coverage(dict(needles={}), chunks_of(c["lens"], c["hkv"], c["sq"], c["mpl"],
                                                        _ctas()), page)["long_chunk"]
                   for c in CASES if c["page"] == page), page


@pytest.mark.parametrize("ci", [0, 9, 19], ids=lambda i: case_id(CASES[i]))
def test_decode_bf16_exact_task_map_sources(hpc, ci):
    """CPU-assigned map, no map (scheduled inside the call with min_process_len 512), lengths
    without the new tokens: each graded against the schedule it runs."""
    c = CASES[ci]
    d, ch = build(c, _ctas(), device="cuda")
    sq, hkv, tag = c["sq"], c["hkv"], f"decode bf16 {case_id(c)}"
    _report(f"{tag} tm=cpu", _run(hpc, d, sq, hkv, c["mpl"], "cpu"), d, sq, ch)
    _report(f"{tag} new_kv_included=False", _run(hpc, d, sq, hkv, c["mpl"], new_kv_included=False),
            d, sq, ch)
    ch512 = chunks_of(c["lens"], hkv, sq, 512, _ctas())
    _report(f"{tag} tm=None", _run(hpc, d, sq, hkv, 512, None), d, sq, ch512)


@pytest.mark.parametrize("lens", [[1], [5, 5, 5], ["p-1", "p", "p+1", 127, 128, 129, 255, 256, 257],
                                  [40000], [129] * 5, [131] * 37], ids=str)
@pytest.mark.parametrize("sq", [1, 4])
@pytest.mark.parametrize("page", [16, 64])
def test_decode_bf16_exact_edge_lengths(hpc, lens, sq, page):
    """A single token, lengths equal to sq, page +- 1, tile edges, one request split over every
    CTA (min_process_len 64), many short requests; needles."""
    lens = [{"p-1": page - 1, "p": page, "p+1": page + 1}.get(n, n) for n in lens]
    lens = [max(int(n), sq) for n in lens]
    for mpl in (64, 1024):
        ch = chunks_of(lens, 2, sq, mpl, _ctas())
        d = make_decode_bf16_exact_inputs("needle", lens, sq, 2, 8, page, chunks=ch, seed=7,
                                          device="cuda")
        _report(f"decode bf16 edge {lens[:3]} sq{sq} bs{page} mpl{mpl}",
                _run(hpc, d, sq, 2, mpl), d, sq, ch)


@pytest.mark.parametrize("page", [16, 32, 64])
def test_rope_store_feeds_bf16_decode(hpc, page):
    """A cache written by rope_norm_store_kv in decode mode (its pages of `page` tokens, NHD,
    tails zeroed) and its rotated q, read by attention_decode_bf16."""
    hq, hkv, B, mtp = 32, 8, 6, 1
    sq = mtp + 1
    d = sr.make_inputs(B, False, mtp, hq, hkv, 128, kv_block_size=page, seed=page,
                       max_num_kv_blocks=160, pad_decode=False)
    c = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in d.items()}
    q = hpc.rope_norm_store_kv(c["kcache"], c["vcache"], c["qkv"], c["cos_sin"], c["num_seqlen"],
                               c["q_index"], c["kv_indices"], False)
    lens = c["num_seqlen"]
    blocks = c["kv_indices"].clamp_min(0).contiguous()
    dd = dict(q=q, kvcache=torch.stack([c["kcache"], c["vcache"]], 1), block_ids=blocks,
              kv_lens_total=lens)
    tm = hpc.get_attention_decode_task_workspace(B, int(lens.max()), hkv, 64)
    hpc.assign_attention_decode_task(lens, tm, hkv, sq, True, 64)
    y = hpc.attention_decode_bf16(q, c["kcache"], c["vcache"], blocks, lens, mtp=mtp,
                                  new_kv_included=True, task_map=tm).cpu()
    ch = chunks_of(lens.cpu().tolist(), hkv, sq, 64, _ctas())
    _report(f"decode bf16 after rope store bs{page}", y, dd, sq, ch)
