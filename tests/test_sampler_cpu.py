"""Fused sampler without a GPU: the numpy Philox against the Random123 known answers, the uniform
mapping, the registered schemas, and that the GPU test's inputs expose every oracle mutation and
clear the rounding margins."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import sampler as osm
from synth import sampler as ss

REPO = Path(__file__).resolve().parents[1]


@pytest.mark.parametrize("ctr,key,expect", [
    ([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
    ([0xffffffff] * 4, [0xffffffff] * 2, [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
    ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0],
     [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]),
])
def test_philox_known_answers(ctr, key, expect):
    out = osm.philox4x32_10(np.array(ctr, np.uint32), np.array(key, np.uint32))
    assert [int(v) for v in out] == expect


def test_uniform_strictly_inside_unit_interval():
    x = np.array([0, 1, 511, 512, 0x7fffffff, 0xfffffe00, 0xffffffff], np.uint32)
    x = np.concatenate([x, np.random.default_rng(0).integers(0, 2 ** 32, 100000, dtype=np.uint64)
                        .astype(np.uint32)])
    u = osm.uniform_from_bits(x)
    assert u.dtype == np.float32 and (u > 0).all() and (u < 1).all()
    assert u.min() == np.float32(2.0 ** -24) and u.max() == np.float32(1 - 2.0 ** -24)
    assert np.isfinite(osm.gumbel_from_uniform(u)).all()


def test_schemas_and_exports(hpc):
    stored = json.loads((REPO / "tests" / "golden" / "reference_schemas.json").read_text())
    for name in ("fused_sampler", "fused_sampler_temperature_sample"):
        schema = str(getattr(torch.ops.hpc, name).default._schema).replace("hpc::", "", 1)
        assert schema == stored[name]
    assert "fused_sampler" in hpc.__all__ and "SoftmaxPolicy" in hpc.__all__
    assert [int(p) for p in hpc.SoftmaxPolicy] == [0, 1, 2]
    assert [p.name for p in hpc.SoftmaxPolicy] == ["NONE", "BEFORE_TOPK", "AFTER_TOPK"]


# The mutation checks run on the GPU test's own cases (synth.sampler.FULL_GRID / FAST_GRID) up to
# B = 64; the B = 512 cases are left out only to keep the CPU suite short.
FULL_CASES = [c for c in ss.FULL_GRID if c[1] <= 64]
FAST_CASES = [c for c in ss.FAST_GRID if c[1] <= 64]


def _full(case, mutations=()):
    n = case["np"]
    kw = {k: v for k, v in n.items() if k not in ("store", "V", "noise")}
    return osm.fused_sampler(n["store"], n["V"], noise=n["noise"], mutations=mutations, **kw)


def _fast(case, mutations=()):
    n = case["np"]
    return osm.temperature_sample(n["store"], n["V"], temperature=n["temperature"], noise=n["noise"],
                                  draft_token_ids=n["draft_token_ids"], mutations=mutations)


@pytest.fixture(scope="module")
def full_cases():
    # building a case redraws noise until every row clears the margins, and raises if one cannot
    return [ss.full_case(*c) for c in FULL_CASES]


@pytest.fixture(scope="module")
def fast_cases():
    return [ss.fast_case(*c) for c in FAST_CASES]


@pytest.fixture(scope="module")
def full_results(full_cases):
    return [_full(c) for c in full_cases]


@pytest.mark.parametrize("mutation", [m for m in osm.MUTATIONS if m != "draft_ignored"])
def test_full_path_inputs_expose_mutation(full_cases, full_results, mutation):
    """Each mutation changes a token (or, for the mask-addressing ones, a token or the written mask)
    on at least one row of the GPU test's full-path cases."""
    for case, (tok, mask) in zip(full_cases, full_results):
        tok_m, mask_m = _full(case, (mutation,))
        if (tok != tok_m).any():
            return
        if mutation in ("mask_bit_msb", "mask_row_b") and not np.array_equal(mask, mask_m):
            return
    pytest.fail(f"no full-path case of the GPU grid exposes {mutation}")


@pytest.mark.parametrize("mutation", ["draft_ignored", "tie_larger_id", "temperature_ignored",
                                      "stride_ignored"])
def test_fast_path_inputs_expose_mutation(fast_cases, mutation):
    assert any((_fast(c) != _fast(c, (mutation,))).any() for c in fast_cases), mutation


def test_full_path_rows_clear_margins(full_cases):
    for case in full_cases:
        n = case["np"]
        kw = {k: v for k, v in n.items() if k not in ("store", "V", "noise")}
        for b in range(n["store"].shape[0]):
            tp, gap = ss.full_row_margins(n["store"], n["V"], kw, n["noise"], b)
            assert tp >= ss.MARGIN and gap >= ss.MARGIN, (b, case["fams"][b], tp, gap)


def test_fast_path_rows_clear_margins(fast_cases):
    for case in fast_cases:
        n = case["np"]
        B = n["store"].shape[0]
        t = np.broadcast_to(np.asarray(n["temperature"], np.float32), (B,))
        for b in range(B):
            gap = osm.fast_row_gap(n["store"][b, :n["V"]], t[b], n["noise"][b], int(n["draft_token_ids"][b]))
            assert gap >= ss.MARGIN, (b, case["fams"][b], gap)


def test_fast_path_cases_have_greedy_rows(fast_cases):
    """The grid holds rows with t = 0, t < 0 and t = NaN, all of which take the plain argmax."""
    t = np.concatenate([np.atleast_1d(c["np"]["temperature"]) for c in fast_cases])
    assert (t == 0).any() and (t < 0).any() and np.isnan(t).any()


def test_builder_raises_when_margins_cannot_be_met():
    noise = np.zeros((1, 64), np.float32)
    with pytest.raises(ValueError, match="rounding decision"):
        ss._redraw_until(lambda: False, noise, 0, np.random.default_rng(0), "row 0", tries=3)
