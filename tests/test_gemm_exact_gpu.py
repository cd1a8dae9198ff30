"""The route GEMM and the stand-alone grouped FP8 GEMMs held element by element to the fp64 oracle
of oracle/gemm_exact.py, on the inputs of synth/gemm_exact.py.

Each graded run prints one line `GEMM <tag> worst_err/B=... acc/E>=...` (pytest -s). For the route
GEMM's fp32 output acc/E is the measured accumulation error over the model's E (the two numbers are
the same there); for bf16 outputs it is moe_exact.accumulation_probe's lower bound."""
import pytest
import torch

from oracle import gemm_exact as ge, moe_exact as ox
from synth import gemm_exact as sg

pytestmark = pytest.mark.gpu

SPLITS = (1, 2, 4, 8)
GUARD_ROWS = 2


def _cuda(d):
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in d.items()}


def _route_rows(c, d):
    return torch.unique(torch.cat([ge.route_rows(c["m"], c["n"], c["k"]), d["cancel_rows"]]))


def _line(tag, worst, acc):
    print(f"GEMM {tag} worst_err/B={worst:.3g} acc/E>={acc:.3g}")


# ------------------------------------------------------------------------------------------------
# route GEMM
# ------------------------------------------------------------------------------------------------
ROUTE_IDS = [sg.route_tag(c) for c in sg.ROUTE_CASES]


@pytest.mark.parametrize("ci", range(len(sg.ROUTE_CASES)), ids=ROUTE_IDS)
def test_route_public_op(hpc, ci):
    """hpc.gemm_bf16xfp32 with use_splitk both ways; the bound takes the split the op selects."""
    c = sg.ROUTE_CASES[ci]
    d = sg.make_route_inputs(c)
    dc = _cuda(d)
    rows = _route_rows(c, d)
    for use_splitk in (False, True):
        split = hpc._ffi.lib.hpc_gemm_bf16xfp32_select_splitk(c["m"], c["n"], c["k"], int(use_splitk))
        y, B, E = ge.route_exact(d["x"], d["w_high"], d["w_low"], d["scale"], split, rows)
        for fp32_out in (True, False):
            out = hpc.gemm_bf16xfp32(dc["x"], dc["w_high"], dc["w_low"], d["scale"], fp32_out, use_splitk)
            assert out.dtype == (torch.float32 if fp32_out else torch.bfloat16)
            assert out.shape == (c["m"], c["n"])
            worst, acc = ge.check_route(out[rows.cuda()].cpu(), y, B, E, fp32_out, ROUTE_IDS[ci])
            _line(f"route/op {ROUTE_IDS[ci]} splitk={int(use_splitk)} split={split} "
                  f"{'fp32' if fp32_out else 'bf16'}", worst, acc)


@pytest.mark.parametrize("ci", range(len(sg.ROUTE_CASES)), ids=ROUTE_IDS)
def test_route_c_entry_every_split(hpc, ci):
    """hpc_gemm_bf16xfp32_async at split 1, 2, 4 and 8 into a NaN-filled buffer with guard rows
    before and after the output (its row stride is n, so those are the only addresses outside it):
    every output element written and within the bound, every guard element still NaN, and repeated
    calls bit-identical."""
    lib, ffi = hpc._ffi.lib, hpc._ffi
    c = sg.ROUTE_CASES[ci]
    m, n, k = c["m"], c["n"], c["k"]
    d = sg.make_route_inputs(c)
    dc = _cuda(d)
    rows = _route_rows(c, d)
    stream = ffi.stream_of(dc["x"])
    for split in SPLITS:
        y, B, E = ge.route_exact(d["x"], d["w_high"], d["w_low"], d["scale"], split, rows)
        idle = sum(1 for *_, st in ge.route_splits(k, split) if st == 0)
        for fp32_out in (True, False):
            outs = []
            for _ in range(2):
                buf = torch.full(((m + 2 * GUARD_ROWS) * n,), float("nan"), device="cuda",
                                 dtype=torch.float32 if fp32_out else torch.bfloat16)
                view = buf[GUARD_ROWS * n:(GUARD_ROWS + m) * n].view(m, n)
                ffi.check(lib.hpc_gemm_bf16xfp32_async(
                    ffi.ptr(view), None, None, ffi.ptr(dc["x"]), ffi.ptr(dc["w_high"]),
                    ffi.ptr(dc["w_low"]), m, n, k, float(d["scale"]), int(fp32_out), split, 128, 1, 0,
                    stream), "gemm_bf16xfp32")
                outs.append(buf)
            torch.cuda.synchronize()
            buf = outs[0]
            assert torch.isnan(buf[:GUARD_ROWS * n]).all() and torch.isnan(buf[(GUARD_ROWS + m) * n:]).all(), \
                f"split {split}: a guard element was written"
            view = buf[GUARD_ROWS * n:(GUARD_ROWS + m) * n].view(m, n)
            unwritten = torch.isnan(view)
            assert not unwritten.any(), (f"split {split}: {int(unwritten.sum())} output elements not "
                                         f"written, first row {int(unwritten.any(1).nonzero()[0])}")
            bits = torch.int32 if fp32_out else torch.int16
            assert torch.equal(outs[0].view(bits), outs[1].view(bits)), f"split {split}: repeated calls differ"
            worst, acc = ge.check_route(view[rows.cuda()].cpu(), y, B, E, fp32_out, ROUTE_IDS[ci])
            _line(f"route/c {ROUTE_IDS[ci]} split={split} idle_ctas={idle} "
                  f"{'fp32' if fp32_out else 'bf16'}", worst, acc)


# ------------------------------------------------------------------------------------------------
# grouped FP8 GEMMs
# ------------------------------------------------------------------------------------------------
def _in_group(seqlens, cu, M):
    gi, _ = ge.group_rows(seqlens, cu)
    inside = torch.zeros(M, dtype=torch.bool)
    inside[:gi.numel()] = gi >= 0
    return inside


def _check_layout(out, seqlens, cu, tag):
    """Rows outside every group still NaN; every row of every group written."""
    inside = _in_group(seqlens, cu, out.size(0))
    assert torch.isnan(out[~inside].float()).all(), f"{tag}: a row outside every group was written"
    assert not torch.isnan(out[inside].float()).any(), f"{tag}: a row of a group was not written"


def _grade(out, y, B, rows, tag):
    if rows.numel() == 0:
        _line(tag + " (no rows)", 0.0, 0.0)
        return
    got = out[rows]
    worst = ox.check_down(got, y, B, tag)
    acc = ox.accumulation_probe(got, y, B, tag)
    _line(tag, worst, acc)


def _sched_dummies(G):
    # the reference's host-side tile tables: accepted and ignored by the device-scheduled kernel
    return torch.zeros(G, dtype=torch.int32, device="cuda"), torch.zeros(G + 1, dtype=torch.int32, device="cuda")


def _bits(t):
    return t.contiguous().view(torch.int16)


@pytest.mark.parametrize("case", sg.PERTENSOR_CASES, ids=[c[0] for c in sg.PERTENSOR_CASES])
def test_pertensor_entries(hpc, case):
    """group_gemm_pertensor_fp8 and group_gemm_fp8 into a NaN-filled output (bit-identical), and
    group_gemm_fp8_cp_async / group_gemm_fp8_scatter_cp_async (identity indices) on the same problem."""
    d = sg.make_pertensor_case(case)
    dc = _cuda(d)
    M, N, K = d["x"].size(0), d["w"].size(1), d["x"].size(1)
    G = d["w"].size(0)
    avg = max(1, int(d["seqlens"].sum()) // G)
    outs = []
    for op in (hpc.group_gemm_pertensor_fp8, hpc.group_gemm_fp8):
        o = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device="cuda")
        r = op(dc["x"], dc["w"], dc["seqlens"], dc["cu_seqlens"], dc["y_scale"],
               num_seq_per_group_avg=avg, output=o)
        assert r.data_ptr() == o.data_ptr()
        outs.append(o.cpu())
    assert torch.equal(_bits(outs[0]), _bits(outs[1])), "group_gemm_fp8 differs from group_gemm_pertensor_fp8"
    out = outs[0]
    _check_layout(out, d["seqlens"], d["cu_seqlens"], case[0])
    rows = ge.rows_to_check(d["seqlens"], d["cu_seqlens"], N, K)
    if rows.numel():
        y, B, _ = ge.grouped_pertensor_exact(d["x"], d["w"], d["seqlens"], d["cu_seqlens"], d["y_scale"], rows)
    else:
        y = B = None
    _grade(out, y, B, rows, f"pertensor {case[0]}")
    inside = _in_group(d["seqlens"], d["cu_seqlens"], M)
    tiles, cu_tiles = _sched_dummies(G)
    cp = torch.ops.hpc.group_gemm_fp8_cp_async(dc["x"], dc["w"], dc["y_scale"], dc["seqlens"],
                                               dc["cu_seqlens"], tiles, cu_tiles, False).cpu()
    assert torch.equal(_bits(cp[inside]), _bits(out[inside])), "cp_async differs from the per-tensor GEMM"
    if not d["gapped"]:
        ident = torch.arange(M, dtype=torch.int32, device="cuda")
        sc = torch.ops.hpc.group_gemm_fp8_scatter_cp_async(dc["x"], dc["w"], dc["y_scale"], ident,
                                                           dc["seqlens"], dc["cu_seqlens"], tiles,
                                                           cu_tiles, False).cpu()
        assert torch.equal(_bits(sc[inside]), _bits(cp[inside])), "scatter (identity) differs from cp_async"


@pytest.mark.parametrize("case", sg.SCATTER_CASES, ids=[c[0] for c in sg.SCATTER_CASES])
def test_scatter_entry(hpc, case):
    """group_gemm_fp8_scatter_cp_async over a pool larger than m with reversed and repeated row
    indices, the pool's last row, and indices -7, -1, pool_rows and pool_rows + 5, which the gather
    clamps to the first and last pool row (the documented behaviour: never read outside the pool)."""
    d = sg.make_scatter_case(case)
    dc = _cuda(d)
    G = d["w"].size(0)
    P = d["pool"].size(0)
    tiles, cu_tiles = _sched_dummies(G)
    out = torch.ops.hpc.group_gemm_fp8_scatter_cp_async(dc["pool"], dc["w"], dc["y_scale"],
                                                        dc["row_indices"], dc["seqlens"],
                                                        dc["cu_seqlens"], tiles, cu_tiles, False).cpu()
    compact = d["pool"][ge.scatter_rows(d["row_indices"], P)]
    cp = torch.ops.hpc.group_gemm_fp8_cp_async(compact.cuda(), dc["w"], dc["y_scale"], dc["seqlens"],
                                               dc["cu_seqlens"], tiles, cu_tiles, False).cpu()
    assert torch.equal(_bits(out), _bits(cp)), "scatter differs from cp_async on the gathered rows"
    rows = ge.rows_to_check(d["seqlens"], d["cu_seqlens"], d["w"].size(1), compact.size(1))
    y, B, _ = ge.grouped_pertensor_exact(compact, d["w"], d["seqlens"], d["cu_seqlens"], d["y_scale"], rows)
    _grade(out, y, B, rows, f"scatter {case[0]}")


def _blockwise_run(hpc, d, xscale_t_cuda, tag):
    dc = _cuda(d)
    M, N = d["x"].size(0), d["w"].size(1)
    o = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device="cuda")
    r = hpc.group_gemm_blockwise_fp8(dc["x"], dc["w"], dc["seqlens"], dc["cu_seqlens"], xscale_t_cuda,
                                     dc["w_scale"], num_seq_per_group_avg=d["avg"], output=o)
    assert r.data_ptr() == o.data_ptr()
    out = o.cpu()
    _check_layout(out, d["seqlens"], d["cu_seqlens"], tag)
    return out


@pytest.mark.parametrize("case", sg.BLOCKWISE_CASES, ids=[c[0] for c in sg.BLOCKWISE_CASES])
def test_blockwise_entry(hpc, case):
    """group_gemm_blockwise_fp8 with NaN in every unused activation-scale column and in the kpad4
    padding of w_scale, into a NaN-filled output."""
    d = sg.make_blockwise_case(case)
    out = _blockwise_run(hpc, d, d["xscale_t"].cuda(), case[0])
    rows = ge.rows_to_check(d["seqlens"], d["cu_seqlens"], d["w"].size(1), d["x"].size(1),
                            granule=d["granule"])
    y, B, _ = ge.grouped_blockwise_exact(d["x"], d["w"], d["seqlens"], d["cu_seqlens"], d["xscale_t"],
                                         d["w_scale"], d["granule"], rows)
    _grade(out, y, B, rows, f"blockwise {case[0]} granule={d['granule']}")


@pytest.mark.parametrize("avg", sg.ROUNDTRIP_AVGS)
def test_deepep_round_trip(hpc, avg):
    """Row-major scales of a gapped (DeepEP) layout -> reformat_x_scale -> group_gemm_blockwise_fp8
    at the same avg: the reformat output equals reformat_layout bit for bit (NaN where unwritten),
    and the GEMM reading it is within the oracle's bound."""
    d = sg.make_roundtrip_case(avg)
    KB, M = d["x"].size(1) // 128, d["x"].size(0)
    xs = torch.full((KB, M), float("nan"), device="cuda")
    r = hpc.reformat_x_scale(d["x_scale"].cuda(), d["seqlens"].cuda(), d["cu_seqlens"].cuda(), avg,
                             output=xs)
    assert r.data_ptr() == xs.data_ptr()
    want = ge.reformat_layout(d["x_scale"], d["seqlens"], d["cu_seqlens"], d["granule"])
    got = xs.cpu()
    assert torch.equal(torch.isnan(got), torch.isnan(want)), f"avg {avg}: reformat wrote the wrong columns"
    assert torch.equal(got.nan_to_num(), want.nan_to_num()), f"avg {avg}: reformat values differ"
    out = _blockwise_run(hpc, d, xs, f"roundtrip avg={avg}")
    rows = ge.rows_to_check(d["seqlens"], d["cu_seqlens"], d["w"].size(1), d["x"].size(1),
                            granule=d["granule"])
    y, B, _ = ge.grouped_blockwise_exact(d["x"], d["w"], d["seqlens"], d["cu_seqlens"], want,
                                         d["w_scale"], d["granule"], rows)
    _grade(out, y, B, rows, f"roundtrip avg={avg} granule={d['granule']}")
