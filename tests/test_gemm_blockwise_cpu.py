"""CPU checks of oracle/gemm_blockwise.py on the inputs of synth/gemm_blockwise.py (no GPU needed).

An fp32 emulation of the dense blockwise FP8 GEMM must pass the per-element check on every case of
the GPU grid's synthetic cases, and each named bug planted in the emulation must fail it on at least
one of them. The quantiser's restatement must be bit-exact on its own special blocks, and each named
quantiser bug must change codes or scales. `pytest -s` prints, per bug, the cases that catch it."""
import functools

import pytest
import torch

from oracle import gemm_blockwise as ob
from synth import gemm_blockwise as sb

IDS = [sb.tag(c) for c in sb.CASES]


@functools.lru_cache(maxsize=None)
def _oracle(ci):
    c = sb.CASES[ci]
    d = sb.make_inputs(c)
    rows = torch.unique(torch.cat([ob.rows_to_check(c["m"], c["n"], c["k"]), d["cancel_rows"]]))
    y, B, _ = ob.gemm_exact(d["x"], d["xs"], d["w"], d["ws"], c["split"], rows)
    return rows, y, B


def _run(ci, bug=None):
    """Grade the emulation; None if it passes, else the failure message."""
    c = sb.CASES[ci]
    d = sb.make_inputs(c)
    rows, y, B = _oracle(ci)
    out = ob.gemm_emulate(d["x"], d["xs"], d["w"], d["ws"], c["split"], rows, bug)
    try:
        ob.check(out, y, B, IDS[ci])
    except AssertionError as e:
        return str(e)
    return None


@pytest.mark.parametrize("ci", range(len(sb.CASES)), ids=IDS)
def test_emulation_passes(ci):
    assert _run(ci) is None


@pytest.mark.parametrize("bug", ob.GEMM_BUGS)
def test_every_gemm_bug_is_caught(bug):
    caught = [IDS[ci] for ci in range(len(sb.CASES)) if _run(ci, bug) is not None]
    print(f"GEMM bug {bug}: caught by {caught}")
    assert caught, f"simulated bug {bug} passes every case"


def test_enough_bugs():
    assert len(ob.GEMM_BUGS) + len(ob.QUANT_BUGS) >= 10


def test_cases_cover_every_split_and_edge():
    assert {c["split"] for c in sb.CASES} == {1, 2, 4, 8}
    assert any(c["n"] % 128 for c in sb.CASES) and any(c["m"] % 128 for c in sb.CASES)
    assert any(c["k"] == 128 for c in sb.CASES)
    for s in (2, 4, 8):
        assert any(c["split"] == s and (c["k"] // 128) % s for c in sb.CASES)
    assert any(sb.make_inputs(c)["cancel_rows"].numel() for c in sb.CASES)


def test_inputs_hold_every_code_and_null_space_rows_cancel():
    for c in sb.CASES:
        assert torch.unique(sb.make_inputs(c)["w"].view(torch.uint8)).numel() == 254
    assert torch.unique(sb.make_inputs(sb.CASES[0])["x"].view(torch.uint8)).numel() == 254
    c = sb.CASES[4]
    d = sb.make_inputs(c)
    rows = d["cancel_rows"]
    y, _, E = ob.gemm_exact(d["x"], d["xs"], d["w"], d["ws"], c["split"], rows)
    _, _, E0 = ob.gemm_exact(d["x"], d["xs"], d["w"], d["ws"], 1, rows)
    S = (E0 / ob.BLOCK_ACC_EPS)  # >= sum_kb |f| S_kb
    assert float((y.abs() / S).max()) < 2.0 ** -6


def test_split_shares_are_contiguous_and_cover_k():
    for k in (128, 640, 1152, 2176):
        for split in (1, 2, 4, 8):
            sh = ob.splits(k, split)
            assert sh[0][0] == 0 and sh[-1][1] == k // 128
            assert all(a[1] == b[0] for a, b in zip(sh, sh[1:]))


# ------------------------------------------------------------------------------------------------
# quantiser
# ------------------------------------------------------------------------------------------------
def test_quant_matches_a_float64_restatement():
    """The fp32 restatement against fp64 arithmetic rounded where the kernel rounds."""
    x = sb.quant_input(37, 640, seed=3)
    q, sc = ob.quant(x)
    v = x.double()
    amax = v.view(37, 5, 128).abs().amax(-1)
    sc64 = (amax / 448.0).float()
    assert torch.equal(sc.view(torch.int32), sc64.contiguous().view(torch.int32))
    inv = (1.0 / (sc64 + 1e-8)).double()  # fp32 add and divide, as the kernel
    prod = (v.view(37, 5, 128) * inv[..., None]).float().view(37, 640)  # exact product, one rounding
    want = prod.clamp(-448, 448).to(torch.float8_e4m3fn)
    assert torch.equal(q.view(torch.uint8), want.view(torch.uint8))


def test_quant_is_the_masked_quantiser_without_silu_mul():
    """The restatement is the blockwise step of oracle/masked_act.py's masked quantiser (which the
    golden fixtures pin): applied to silu(gate) * up it gives that oracle's codes and scales."""
    from oracle import masked_act as oma

    g = torch.Generator().manual_seed(7)
    gu = (torch.randn((48, 2 * 640), generator=g) * 3).to(torch.bfloat16)
    gu[:4, :640] = 0.0  # all-zero blocks
    q, sc = oma.masked_act_mul_and_blockwise_quant(gu)
    assert ob.quant_mismatch(*ob._quant(oma._silu_mul(gu)), q, sc) == (0, 0)


def test_quant_special_blocks():
    x = sb.quant_input(64, 1024, seed=1)
    q, sc = ob.quant(x)
    blocks = x.float().view(64, 8, 128)
    zero = (blocks == 0).all(-1)
    assert zero.any() and (sc[zero] == 0).all()
    assert (q.view(torch.uint8).view(64, 8, 128)[zero] & 0x7F == 0).all()
    tiny = (blocks.abs().amax(-1) < 2e-6) & ~zero
    assert tiny.any()
    big = blocks.abs().amax(-1) > 1e38
    assert big.any()
    assert torch.isfinite(sc).all()
    assert ((q.view(torch.uint8) & 0x7F) != 0x7F).all()


@pytest.mark.parametrize("bug", ob.QUANT_BUGS)
def test_every_quant_bug_is_caught(bug):
    x = sb.quant_input(64, 1024, seed=1)
    q, sc = ob.quant(x)
    bq, bs = ob.quant_emulate(x, bug)
    assert sum(ob.quant_mismatch(bq, bs, q, sc)) > 0, bug


def test_strided_quant_input():
    x = sb.quant_input(5, 256, seed=2, ld=264)
    assert x.stride(0) == 264 and not x.is_contiguous()
    q, sc = ob.quant(x)
    q2, sc2 = ob.quant(x.contiguous())
    assert ob.quant_mismatch(q, sc, q2, sc2) == (0, 0)
