"""The exact-reference check of bf16 paged decode can tell (CPU only).

CASES is the case list tests/test_decode_bf16_exact_gpu.py runs on the GPU: every page size
(16, 32, 64) meets both layouts, both input families of
synth.attention_exact.make_decode_bf16_exact_inputs and every query-row count of the kernel's
instantiations (4, 8, 12, 16, 20, 24, 32 rows per kv head). For each case the lossy oracle (P
rounded to bf16 against the row maximum) passes both parts of oracle.attention_exact.grade
against oracle.prefill_bf16.decode_exact, and every simulated kernel bug of
oracle.prefill_bf16.DECODE_MUTATIONS that the case can express fails one of them. The split-k
chunks come from the schedule the GPU run uses (oracle.taskmap with one CTA per SM of an H100
SXM), and the case list is checked to exercise what it claims: chunks longer than 32 pages,
needles past the first chunk, single-chunk and multi-chunk pairs in one call.
"""
import pytest
import torch

from oracle import attention_exact as ox
from oracle import prefill_bf16 as ob
from oracle import taskmap as otm
from synth.attention_exact import make_decode_bf16_exact_inputs

NUM_CTAS = 132  # sm_count * _CTA_PER_SM (hpc/attention.py) on an H100 SXM
PAGES = (16, 32, 64)

# rows per kv head -> (hkv, hq, sq) choices; group 4 or 8, sq 1-4 and 5 with group 4
_ROWS = {
    4: [(1, 4, 1), (2, 8, 1)],
    8: [(1, 8, 1), (4, 32, 1), (8, 64, 1), (1, 4, 2)],
    12: [(1, 4, 3), (2, 8, 3)],
    16: [(2, 8, 4), (4, 32, 2), (1, 8, 2)],
    20: [(1, 4, 5), (2, 8, 5)],
    24: [(1, 8, 3), (4, 32, 3), (8, 64, 3)],
    32: [(4, 32, 4), (1, 8, 4), (8, 64, 4)],
}


def _cases():
    out = []
    for pi, page in enumerate(PAGES):
        for ri, (rows, opts) in enumerate(_ROWS.items()):
            hkv, hq, sq = opts[pi % len(opts)]
            kind = ("needle", "peaked")[(ri // 2 + pi) % 2]
            out.append(dict(
                page=page, rows=rows, hkv=hkv, hq=hq, sq=sq, kind=kind,
                temp=(1.0, 4.0, 16.0)[(ri + pi) % 3] if kind == "peaked" else 0.0,
                layout=("NHD", "HND")[(ri + pi) % 2],
                # 4096: a chunk spans 32 tiles (> 32 pages); 64: chunks of a few tiles
                mpl=(4096, 64)[(ri // 3 + ri + pi) % 2],
                # ragged: a long request split into chunks, a short one of one tile (single
                # chunk, partial page), a middle one
                lens=[6001 + 29 * ri + 6 * pi, page + 3 + ri, 1001 + 64 * ri],
                seed=100 * pi + ri))
    return out


CASES = _cases()


def case_id(c):
    return (f"bs{c['page']}-{c['layout']}-r{c['rows']}-h{c['hkv']}x{c['hq']}-sq{c['sq']}-"
            f"{c['kind']}{c['temp'] if c['kind'] == 'peaked' else ''}-mpl{c['mpl']}")


def chunks_of(lens, hkv, sq, mpl, num_ctas=NUM_CTAS):
    return otm.pair_chunks(lens, num_ctas, hkv, sq, mpl)


def build(c, num_ctas=NUM_CTAS, device="cpu"):
    """Inputs of case c with needles placed for its schedule; returns (inputs, chunks)."""
    ch = chunks_of(c["lens"], c["hkv"], c["sq"], c["mpl"], num_ctas)
    d = make_decode_bf16_exact_inputs(c["kind"], c["lens"], c["sq"], c["hkv"], c["hq"], c["page"],
                                      temperature=c["temp"], layout=c["layout"], chunks=ch,
                                      seed=c["seed"], device=device)
    return d, ch


def _args(d):
    kv = d["kvcache"].cpu()
    return (d["q"].cpu(), kv[:, 0], kv[:, 1], d["block_ids"].cpu(), d["kv_lens_total"].cpu())


def exact(d, sq, chunks):
    return ob.decode_exact(*_args(d), sq, chunks)


def lossy(d, sq, chunks, mutation=None):
    return ob.decode_exact(*_args(d), sq, chunks, lossy=True, mutation=mutation)[0]


def coverage(d, chunks, page):
    """What one call under `chunks` exercises."""
    n = dict(single=False, multi=False, long_chunk=False, needle_past_first=False)
    for (b, h), ch in chunks.items():
        n["single" if len(ch) == 1 else "multi"] = True
        n["long_chunk"] |= any(ln > 32 * page for _, ln in ch)
        if len(ch) > 1 and (b, h) in d["needles"]:
            n["needle_past_first"] |= any(p >= ch[1][0] for p in d["needles"][(b, h)])
    return n


def mutations_for(c, chunks):
    """The decode mutations case c can express (the others leave its output unchanged)."""
    cov = coverage(dict(needles={}), chunks, c["page"])
    out = []
    for m in ob.DECODE_MUTATIONS:
        if (m == "mtp_rows_swapped" and c["sq"] == 1) or (m == "kv_head_mod" and c["hkv"] == 1):
            continue
        if m == "page_group_wrap" and not cov["long_chunk"]:
            continue
        if m.startswith("chunk_") or m == "lse_natural_log":
            if not cov["multi"]:
                continue
        out.append(m)
    return out


@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_decode_bf16_exact_checks_discriminate(c):
    d, ch = build(c)
    sq = c["sq"]
    y, bound = exact(d, sq, ch)
    ref = lossy(d, sq, ch)
    r = ox.grade(ref, y, bound, ref)
    assert r["ok_a"] and r["ok_b"], f"lossy oracle fails the check: {r}"
    assert r["rel_oracle"] < 0.05, r
    undetected = []
    for m in mutations_for(c, ch):
        rm = ox.grade(lossy(d, sq, ch, m), y, bound, ref)
        if rm["ok_a"] and rm["ok_b"]:
            undetected.append((m, rm))
    assert not undetected, undetected


def test_decode_bf16_cases_cover_what_they_claim():
    """Per page size: a chunk longer than 32 pages (the producer's second group of page ids),
    both min_process_len values, every row count, both layouts and both families; per case:
    single-chunk and multi-chunk pairs in one call, and a needle past the first chunk of a pair."""
    for page in PAGES:
        cs = [c for c in CASES if c["page"] == page]
        assert {c["rows"] for c in cs} == set(_ROWS)
        assert {c["layout"] for c in cs} == {"NHD", "HND"}
        assert {c["kind"] for c in cs} == {"needle", "peaked"}
        assert {c["mpl"] for c in cs} == {64, 4096}
        long_chunk = False
        for c in cs:
            d, ch = build(c)
            cov = coverage(d, ch, page)
            assert cov["single"] and cov["multi"], (case_id(c), cov)
            if c["kind"] == "needle":
                assert cov["needle_past_first"], (case_id(c), cov)
            long_chunk |= cov["long_chunk"]
        assert long_chunk, f"no chunk longer than 32 pages of {page}"
    assert {(c["hkv"], c["hq"]) for c in CASES} == {(1, 4), (1, 8), (2, 8), (4, 32), (8, 64)}
    assert {c["sq"] for c in CASES} == {1, 2, 3, 4, 5}
    for m in ob.DECODE_MUTATIONS:  # every mutation is checked on some case of each page size
        for page in PAGES:
            assert any(m in mutations_for(c, chunks_of(c["lens"], c["hkv"], c["sq"], c["mpl"]))
                       for c in CASES if c["page"] == page), (m, page)


def test_decode_exact_equals_paged_prefill_exact_without_combine():
    """With one chunk per pair decode_exact is paged_exact with cu_seqlens_q = sq * arange(B + 1),
    and a split pair only adds the combine term to the bound."""
    c = CASES[3]
    d, ch = build(c)
    q, k, v, ids, lens = _args(d)
    cu = c["sq"] * torch.arange(lens.numel() + 1)
    y0, b0 = ob.paged_exact(q, k, v, cu, ids, lens)
    one = {key: [(0, int(lens[key[0]]))] for key in ch}
    y1, b1 = ob.decode_exact(q, k, v, ids, lens, c["sq"], one)
    assert torch.equal(y0, y1) and torch.equal(b0, b1)
    y2, b2 = ob.decode_exact(q, k, v, ids, lens, c["sq"], ch)
    assert torch.equal(y0, y2) and bool((b2 >= b0).all()) and bool((b2 > b0).any())
