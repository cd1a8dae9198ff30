"""CPU checks of oracle/gemm_exact.py on the inputs of synth/gemm_exact.py (no GPU needed).

An fp32 emulation of each kernel's arithmetic must pass the per-element check on every case, and
each named bug planted in the emulation must fail it on at least one case that can express it. The
test prints, per bug, the cases that catch it (`pytest -s`). A last group of tests shows which of
these bugs the reference-tolerance checks of tests/test_gemm_gpu.py, test_moe_gpu.py and
test_act_gpu.py let through."""
import functools
import importlib

import pytest
import torch

from oracle import gemm as og, gemm_exact as ge, moe_exact as ox
from synth import gemm_exact as sg

SPLITS = (1, 2, 4, 8)


# ------------------------------------------------------------------------------------------------
# route GEMM
# ------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _route_rows(ci):
    c = sg.ROUTE_CASES[ci]
    d = sg.make_route_inputs(c)
    rows = torch.cat([ge.route_rows(c["m"], c["n"], c["k"]), d["cancel_rows"]])
    return torch.unique(rows)


@functools.lru_cache(maxsize=64)
def _route_oracle(ci, split):
    d = sg.make_route_inputs(sg.ROUTE_CASES[ci])
    return ge.route_exact(d["x"], d["w_high"], d["w_low"], d["scale"], split, _route_rows(ci))


def _route_run(ci, split, fp32_out, bug=None):
    """Grade the emulation; returns None if it passes, else the failure message."""
    d = sg.make_route_inputs(sg.ROUTE_CASES[ci])
    rows = _route_rows(ci)
    out = ge.route_emulate(d["x"], d["w_high"], d["w_low"], d["scale"], split, fp32_out, rows, bug)
    y, B, E = _route_oracle(ci, split)
    try:
        ge.check_route(out, y, B, E, fp32_out)
    except AssertionError as e:
        return str(e)
    return None


@pytest.mark.parametrize("ci", range(len(sg.ROUTE_CASES)),
                         ids=[sg.route_tag(c) for c in sg.ROUTE_CASES])
def test_route_emulation_passes(ci):
    for split in SPLITS:
        for fp32_out in (True, False):
            msg = _route_run(ci, split, fp32_out)
            assert msg is None, (split, fp32_out, msg)


def test_route_cases_cover_the_kernel():
    ks = {c["k"] for c in sg.ROUTE_CASES}
    assert {8, 56, 64, 72, 200, 1000, 4096, 7168} <= ks
    assert {1, 7, 127, 128, 129, 255, 1000, 12303} <= {c["m"] for c in sg.ROUTE_CASES}
    assert {64, 192, 320, 128, 256, 2048, 7168} <= {c["n"] for c in sg.ROUTE_CASES}
    # a case where a whole CTA of the cluster has no K step, at split 4 and at split 8
    for split in (4, 8):
        assert any(steps == 0 for c in sg.ROUTE_CASES for *_, steps in ge.route_splits(c["k"], split))
    # K-step counts that the split does not divide, with every CTA busy
    for split in (2, 4, 8):
        assert any(all(st for *_, st in ge.route_splits(c["k"], split)) and ((c["k"] + 63) // 64) % split
                   for c in sg.ROUTE_CASES)
    # strong cancellation: |y| << S on the planted rows
    d = sg.make_route_inputs(sg.ROUTE_CASES[6])
    rows = d["cancel_rows"]
    X = d["x"][rows].double()
    weff = d["w_high"].double() + d["scale"] * d["w_low"].double()
    y, S = X @ weff.t(), X.abs() @ weff.abs().t()
    assert float((y.abs() / S).max()) < 2e-3


@pytest.mark.parametrize("bug", ge.ROUTE_BUGS)
def test_route_bug_caught(bug):
    catchers, missed = [], []
    for ci, c in enumerate(sg.ROUTE_CASES):
        d = sg.make_route_inputs(c)
        for split in SPLITS:
            for fp32_out in (True, False):
                if not ge.route_bug_expressible(bug, c["m"], c["n"], c["k"], d["scale"], split, fp32_out):
                    continue
                tag = f"{sg.route_tag(c)}/split{split}/{'fp32' if fp32_out else 'bf16'}"
                (catchers if _route_run(ci, split, fp32_out, bug) else missed).append(tag)
    print(f"\nBUG route.{bug}: caught by {len(catchers)} runs, e.g. {catchers[:6]}; "
          f"expressed but not caught by {len(missed)}")
    assert catchers, f"route bug {bug} is caught by no case"


# ------------------------------------------------------------------------------------------------
# grouped FP8 GEMMs
# ------------------------------------------------------------------------------------------------
def _grouped_cases():
    out = []
    for c in sg.PERTENSOR_CASES:
        out.append(("pt", c))
    for c in sg.SCATTER_CASES:
        out.append(("scatter", c))
    for c in sg.BLOCKWISE_CASES:
        out.append(("bw", c))
    for a in sg.ROUNDTRIP_AVGS:
        out.append(("roundtrip", a))
    return out


GROUPED = _grouped_cases()


def _gtag(kind, c):
    return f"roundtrip_avg{c}" if kind == "roundtrip" else c[0]


@functools.lru_cache(maxsize=None)
def _grouped_data(i):
    kind, c = GROUPED[i]
    if kind == "pt":
        return sg.make_pertensor_case(c)
    if kind == "scatter":
        return sg.make_scatter_case(c)
    if kind == "bw":
        return sg.make_blockwise_case(c)
    d = sg.make_roundtrip_case(c)
    # the layout reformat_x_scale writes, with the GEMM's granule
    return dict(d, xscale_t=ge.reformat_layout(d["x_scale"], d["seqlens"], d["cu_seqlens"], d["granule"]))


def _compact_x(d, bug=None):
    if "pool" in d:
        return d["pool"][ge.scatter_rows(d["row_indices"], d["pool"].size(0), bug)]
    return d["x"]


@functools.lru_cache(maxsize=None)
def _grouped_oracle(i):
    d = _grouped_data(i)
    x = _compact_x(d)
    rows = ge.rows_to_check(d["seqlens"], d["cu_seqlens"], d["w"].size(1), x.size(1),
                            granule=d.get("granule"))
    if "y_scale" in d:
        y, B, _ = ge.grouped_pertensor_exact(x, d["w"], d["seqlens"], d["cu_seqlens"], d["y_scale"], rows)
    else:
        y, B, _ = ge.grouped_blockwise_exact(x, d["w"], d["seqlens"], d["cu_seqlens"], d["xscale_t"],
                                             d["w_scale"], d["granule"], rows)
    return rows, y, B


def _grouped_run(i, bug=None):
    d = _grouped_data(i)
    rows, y, B = _grouped_oracle(i)
    if rows.numel() == 0:  # every group empty: nothing to grade here (the GPU test checks no write)
        return None
    x = _compact_x(d, bug)
    out = ge.grouped_emulate(x, d["w"], d["seqlens"], d["cu_seqlens"], rows, y_scale=d.get("y_scale"),
                             xscale_t=d.get("xscale_t"), w_scale=d.get("w_scale"), avg=d.get("avg"),
                             bug=bug)
    try:
        ox.check_down(out, y, B, "grouped")
    except AssertionError as e:
        return str(e)
    return None


@pytest.mark.parametrize("i", range(len(GROUPED)), ids=[_gtag(*c) for c in GROUPED])
def test_grouped_emulation_passes(i):
    assert _grouped_run(i) is None


def _expressible(bug, i):
    kind, _ = GROUPED[i]
    d = _grouped_data(i)
    sl, cu = d["seqlens"], d["cu_seqlens"]
    busy = sl > 0
    x = _compact_x(d)
    blockwise = "y_scale" not in d
    if bug == "yscale_neighbour":
        return not blockwise and sl.numel() > 1 and bool(busy.any())
    if bug == "rows_from_seqlens_prefix":
        prefix = torch.cumsum(sl, 0) - sl
        return bool(((prefix != cu[:-1]) & busy).any())
    if bug == "drop_last_kblock":
        return bool(busy.any())
    if bug == "subnormal_as_normal":
        def sub(t):
            b = t.view(torch.uint8)
            return bool((((b & 0x78) == 0) & ((b & 7) != 0)).any())
        return sub(x) or sub(d["w"])
    if bug == "reformat_granule":
        return blockwise and bool(((ge.pad_base(sl, ge.reformat_granule_old(d["avg"]))
                                    != ge.pad_base(sl, d["granule"])) & busy).any())
    if bug == "wscale_stride_kb":
        return blockwise and d["w_scale"].size(2) != x.size(1) // 128
    if bug == "act_scale_next_row":
        return blockwise and bool(busy.any())
    if bug == "scatter_off_by_one":
        return kind == "scatter"
    raise KeyError(bug)


CATCHERS = {
    # the named cases that must catch each bug (others may too)
    "yscale_neighbour": {"codes_x", "g8_edges", "g8_gapped"},
    "rows_from_seqlens_prefix": {"g8_gapped", "g128_gapped"} | {f"roundtrip_avg{a}" for a in sg.ROUNDTRIP_AVGS},
    "drop_last_kblock": {"codes_x", "g8_edges", "g1_big", "bw_g8_edges"},
    "subnormal_as_normal": {"codes_x", "codes_w"},
    "reformat_granule": {"roundtrip_avg80", "roundtrip_avg110", "roundtrip_avg140"},
    "wscale_stride_kb": {"bw_g8_edges", "bw_g1_k512"},
    "act_scale_next_row": {"bw_g8_edges", "roundtrip_avg5", "roundtrip_avg200"},
    "scatter_off_by_one": {"scatter_edges", "scatter_g8"},
}


@pytest.mark.parametrize("bug", ge.GROUPED_BUGS)
def test_grouped_bug_caught(bug):
    catchers, missed = [], []
    for i, (kind, c) in enumerate(GROUPED):
        if not _expressible(bug, i):
            continue
        (catchers if _grouped_run(i, bug) else missed).append(_gtag(kind, c))
    print(f"\nBUG grouped.{bug}: caught by {catchers}; expressed but not caught by {missed}")
    assert catchers, f"grouped bug {bug} is caught by no case"
    assert CATCHERS[bug] <= set(catchers), CATCHERS[bug] - set(catchers)


def test_grouped_cases_cover_the_kernel():
    every_code = sg.finite_codes().view(torch.uint8)
    assert every_code.numel() == 254
    d = sg.make_pertensor_case(sg.PERTENSOR_CASES[0])
    assert set(d["x"].view(torch.uint8).unique().tolist()) >= set(every_code.tolist())
    # every code at every K position of a block: position of code i walks by 37 (coprime to K)
    pos = d["x"].view(torch.uint8).ne(0).float().argmax(1)
    assert pos.unique().numel() == d["x"].size(1)
    d = sg.make_pertensor_case(sg.PERTENSOR_CASES[1])
    assert set(d["w"].view(torch.uint8).unique().tolist()) >= set(every_code.tolist())
    rows = set()
    for c in sg.PERTENSOR_CASES:
        if isinstance(c[1], list):
            rows |= set(c[1])
    assert {0, 1, 63, 64, 65, 127, 128, 129, 300} <= rows
    gs = {sg.make_pertensor_case(c)["seqlens"].numel() for c in sg.PERTENSOR_CASES}
    assert {1, 8, 128, 512} <= gs
    assert {64, 192, 320, 4096} <= {c[3] for c in sg.PERTENSOR_CASES}
    assert {16, 48, 144, 192, 1008, 7168} <= {c[4] for c in sg.PERTENSOR_CASES}
    # every bucket of the GEMM's granule rule is a round trip
    buckets = [(0, 8), (9, 16), (17, 32), (33, 48), (49, 64), (65, 96), (97, 128), (129, 144),
               (145, 1 << 30)]
    assert all(any(lo <= a <= hi for a in sg.ROUNDTRIP_AVGS) for lo, hi in buckets)
    # scatter: pool larger than m, the pool's last row, and indices that are clamped
    d = sg.make_scatter_case(sg.SCATTER_CASES[0])
    idx, P = d["row_indices"], d["pool"].size(0)
    assert P > idx.numel() and (idx == P - 1).any() and (idx < 0).any() and (idx >= P).any()


def test_reformat_layout_and_granules():
    sl = torch.tensor([3, 0, 5], dtype=torch.int32)
    cu = torch.tensor([0, 8, 16, 24], dtype=torch.int32)
    xs = torch.arange(24 * 2, dtype=torch.float32).view(24, 2)
    lay = ge.reformat_layout(xs, sl, cu, 8)
    assert torch.equal(lay[:, 0:3], xs[0:3].t()) and torch.equal(lay[:, 8:13], xs[16:21].t())
    assert torch.isnan(lay[:, 3:8]).all() and torch.isnan(lay[:, 13:]).all()
    # the old reformat rule and the GEMM's disagree exactly on 65 <= avg <= 144
    differ = [a for a in range(1, 300) if ge.reformat_granule_old(a) != ox.scale_granule(a)]
    assert differ == list(range(65, 145))


def test_library_shares_the_gemm_granule(hpc):
    """reformat_x_scale, the FusedMoE host code and the grouped GEMM take one granule rule."""
    fuse_moe = importlib.import_module("hpc.fuse_moe")
    group_gemm = importlib.import_module("hpc.group_gemm")

    for a in range(0, 400):
        want = ox.scale_granule(a)
        assert group_gemm._scale_tile(a) == want
        assert fuse_moe._aligned_size(a) == want
        assert hpc._ffi.lib.hpc_scale_tile_from_avg(a) == want


# ------------------------------------------------------------------------------------------------
# what the reference-tolerance checks let through
# ------------------------------------------------------------------------------------------------
def _old_route_ok(out, fp32_out, x, w, wh, wl, scale):
    """tests/test_gemm_gpu.py: allclose(rtol 0.08, atol 0.01) against the fp32 matmul with the
    unsplit weight, and for fp32 output relative L2 < 1e-5 against the exact split product."""
    gt = og.gemm_fp32(x, w)
    if not torch.allclose(gt, out.float(), rtol=0.08, atol=0.01):
        return False
    if fp32_out:
        exact = og.gemm_split_exact(x, wh, wl, scale)
        return bool((out.double() - exact).norm() / exact.norm() < 1e-5)
    return True


def test_reference_tolerance_route_misses():
    """On the old grid's shape (m 144, n 192, k 4096, split 4), which route bugs pass the old check
    of the output path that shows them; the new check (test_route_bug_caught) catches all of them."""
    m, n, k, split = 144, 192, 4096, 4
    x, w, wh, wl, scale = og.make_inputs(m, n, k)
    missed = {}
    for bug in ge.ROUTE_BUGS:
        for fp32_out in (True, False):
            if not ge.route_bug_expressible(bug, m, n, k, scale, split, fp32_out):
                continue
            out = ge.route_emulate(x, wh, wl, scale, split, fp32_out, bug=bug)
            if _old_route_ok(out, fp32_out, x, w, wh, wl, scale):
                missed.setdefault(bug, []).append("fp32" if fp32_out else "bf16")
    print(f"\nroute bugs the reference-tolerance checks miss: {missed}")
    for fp32_out in (True, False):
        assert _old_route_ok(ge.route_emulate(x, wh, wl, scale, split, fp32_out), fp32_out,
                             x, w, wh, wl, scale)
    assert missed == {"bf16_truncate": ["bf16"]}, missed


def test_reference_tolerance_grouped_misses():
    """The grouped GEMM bugs that the reference-tolerance checks of test_moe_gpu.py (per-tensor
    rtol 0.08 / atol 0.01 with y_scale ~ U(0, 0.01); blockwise rtol 0.01 / atol 0.05 on randn / 10)
    and test_act_gpu.py (rtol 1e-2 / atol 0.25 with y_scale ~ U(0.5, 1.5)) let through, on their
    input distributions (randn e4m3) at small shapes."""
    g = torch.Generator().manual_seed(41)
    G, n, k = 4, 256, 512
    seqlens = torch.tensor([30, 70, 0, 64], dtype=torch.int32)
    cu = torch.zeros(G + 1, dtype=torch.int32)
    cu[1:] = torch.cumsum(seqlens, 0)
    M = int(cu[-1])
    rows = torch.arange(M)
    x = torch.randn((M, k), generator=g).to(torch.float8_e4m3fn)
    w = torch.randn((G, n, k), generator=g).to(torch.float8_e4m3fn)
    missed = {}
    for tag, ys, rtol, atol in (("moe", torch.rand(G, generator=g) * 0.01, 0.08, 0.01),
                                ("act", torch.rand(G, generator=g) + 0.5, 1e-2, 0.25)):
        gt = torch.cat([(x[cu[i]:cu[i + 1]].float() @ w[i].float().t()) * ys[i] for i in range(G)])
        for bug in ("yscale_neighbour", "drop_last_kblock", "subnormal_as_normal"):
            out = ge.grouped_emulate(x, w, seqlens, cu, rows, y_scale=ys, bug=bug)
            if torch.allclose(out.float(), gt, rtol=rtol, atol=atol):
                missed.setdefault(bug, []).append(f"pertensor/{tag}")
        out = ge.grouped_emulate(x, w, seqlens, cu, rows, y_scale=ys)
        assert torch.allclose(out.float(), gt, rtol=rtol, atol=atol)
    # blockwise (test_moe_gpu.test_group_gemm_blockwise)
    xb = (torch.randn((M, k), generator=g) / 10).to(torch.float8_e4m3fn)
    wb = (torch.randn((G, n, k), generator=g) / 10).to(torch.float8_e4m3fn)
    xs_rows = torch.randn((M, k // 128), generator=g)
    ws = torch.randn((G, n // 128, k // 128 + 4), generator=g)
    avg = 80
    xs_t = ge.reformat_layout(xs_rows, seqlens, cu, ox.scale_granule(avg))
    xs_t = torch.nan_to_num(xs_t, nan=0.0)
    from oracle import moe as om
    gt = om.group_gemm_blockwise(xb, wb, seqlens, cu, xs_rows, ws).float()
    for bug in ("drop_last_kblock", "subnormal_as_normal", "reformat_granule", "wscale_stride_kb",
                "act_scale_next_row"):
        out = ge.grouped_emulate(xb, wb, seqlens, cu, rows, xscale_t=xs_t, w_scale=ws, avg=avg, bug=bug)
        if torch.allclose(out.float().nan_to_num(1e9), gt, rtol=0.01, atol=0.05):
            missed.setdefault(bug, []).append("blockwise")
    print(f"\ngrouped bugs the reference-tolerance checks miss: {missed}")
    assert missed == {"subnormal_as_normal": ["pertensor/moe"]}, missed
