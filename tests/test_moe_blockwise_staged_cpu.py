"""CPU proof of the staged blockwise FusedMoE oracle (oracle/moe_exact.py): every stage passes
against its own emulation of the kernel, and each mutation a wrong kernel could make is rejected.
Also checks that the routed input builder gives O(1) outputs for every routing."""
import pytest
import torch

from oracle import moe_exact as ox
from synth.moe import make_moe_blockwise_routed_inputs

T, K, H, I, E_TOTAL = 175, 8, 640, 384, 32  # avg 43 -> granule 48; kpad4 != K/128 on both GEMMs


def _pipeline(d):
    """Emulated kernel outputs of every stage (all rows), built from the oracle's own arithmetic."""
    E = d["gate_up_weight"].size(0)
    t, k = d["topk_ids"].shape
    r = ox.route(d["topk_ids"], E, d["rank_ep"], d["num_expert_total"])
    rows_total = r["src_token"].numel()
    gran = r["granule"]
    num_padded = (t * k + d["num_expert_total"] * gran + gran - 1) // gran * gran
    gathered = d["x"][r["src_token"]]
    xs_layout = ox.scale_layout(d["x_scale"], r, num_padded)
    allrows = torch.arange(rows_total)
    codes, sc = ox.gateup_emulate(gathered, xs_layout, r, d["gate_up_weight"],
                                  d["gate_up_weight_scale"], allrows)
    di_layout = torch.full((I // 128, num_padded), float("nan"))
    di_layout[:, r["col_of_row"]] = sc
    y, _ = ox.down_exact(codes, di_layout, r, d["down_weight"], d["down_weight_scale"], allrows)
    down_out = y.to(torch.bfloat16)
    o, _ = ox.reduce_exact(down_out, r["topk_pos"], d["topk_scale"], d["shared_output"])
    return dict(r=r, gathered=gathered, xs_layout=xs_layout, codes=codes, di_layout=di_layout,
                down_out=down_out, out=o.to(torch.bfloat16), num_padded=num_padded)


@pytest.fixture(scope="module")
def case():
    d = make_moe_blockwise_routed_inputs(T, K, H, I, E_TOTAL, routing="hot", seed=3)
    return d, _pipeline(d)


@pytest.mark.parametrize("routing,size_ep,rank_ep,t", [("uniform", 1, 0, T), ("hot", 1, 0, T),
                                                       ("sparse", 1, 0, 16),
                                                       ("other_ranks", 4, 2, T)])
def test_builder_outputs_are_order_one(routing, size_ep, rank_ep, t):
    d = make_moe_blockwise_routed_inputs(t, K, H, I, E_TOTAL if routing != "sparse" else 128,
                                         routing=routing, size_ep=size_ep, rank_ep=rank_ep,
                                         shared=routing == "other_ranks", seed=5)
    p = _pipeline(d)
    x = d["x"].float()
    assert (x.abs() >= 2.0 ** -6).all(), "x must be in e4m3's normal range"
    rms = float(p["down_out"].float().pow(2).mean().sqrt())
    assert 0.2 < rms < 5, f"{routing}: Down output rms {rms}"
    rms = float(p["out"].float().pow(2).mean().sqrt())
    assert 0.2 < rms < 5, f"{routing}: output rms {rms}"


# ------------------------------------------------------------------------------------------------
# route
# ------------------------------------------------------------------------------------------------
def _route_got(d, p, layout=None):
    r = p["r"]
    return dict(counts=r["counts"], cu_counts=r["cu"], topk_pos=r["topk_pos"],
                gate_up_input=p["gathered"], gate_up_input_scale=p["xs_layout"] if layout is None else layout)


def _layout_with(d, r, cols, num_padded):
    out = torch.full((H // 128, num_padded + 256), float("nan"))
    out[:, cols] = d["x_scale"][r["src_token"]].t().float()
    return out


def test_route_passes(case):
    d, p = case
    assert p["r"]["granule"] == 48
    ox.check_route(p["r"], d["x"], d["x_scale"], _route_got(d, p))


def test_route_rejects_granule_64(case):
    d, p = case
    r = p["r"]
    padded = (r["counts"] + 63) // 64 * 64
    base = torch.zeros_like(r["pad_base"])
    base[1:] = torch.cumsum(padded, 0)[:-1]
    cols = base[r["expert_of_row"]] + r["local_index"]
    with pytest.raises(AssertionError, match="layout"):
        ox.check_route(r, d["x"], d["x_scale"], _route_got(d, p, _layout_with(d, r, cols, p["num_padded"])))


def test_route_rejects_last_pad_base_plus_4(case):
    d, p = case
    r = p["r"]
    last = int((r["counts"] > 0).nonzero().max())
    cols = r["col_of_row"] + 4 * (r["expert_of_row"] == last)
    with pytest.raises(AssertionError, match="layout"):
        ox.check_route(r, d["x"], d["x_scale"], _route_got(d, p, _layout_with(d, r, cols, p["num_padded"])))


# ------------------------------------------------------------------------------------------------
# Gate-Up
# ------------------------------------------------------------------------------------------------
def _gateup(d, p, codes=None, di_layout=None):
    r = p["r"]
    rows = ox.rows_to_check(r, seed=1)
    return ox.check_gateup(p["gathered"], p["xs_layout"], r, d["gate_up_weight"],
                           d["gate_up_weight_scale"], rows,
                           p["codes"] if codes is None else codes,
                           p["di_layout"] if di_layout is None else di_layout)


def test_gateup_passes(case):
    d, p = case
    st = _gateup(d, p)
    assert st["flips"] == 0


def test_gateup_rejects_scale_from_next_k_block(case):
    d, p = case
    r = p["r"]
    row = int(ox.rows_to_check(r, seed=1)[5])
    xs = p["xs_layout"].clone()
    c = int(r["col_of_row"][row])
    xs[0, c] = xs[1, c]
    rows = torch.tensor([row])
    codes, sc = ox.gateup_emulate(p["gathered"], xs, r, d["gate_up_weight"],
                                  d["gate_up_weight_scale"], rows)
    mc, ml = p["codes"].clone(), p["di_layout"].clone()
    mc[row] = codes[0]
    ml[:, c] = sc[:, 0]
    with pytest.raises(AssertionError, match="gate-up"):
        _gateup(d, p, mc, ml)


def _far_element(d, p, row):
    """A column of `row` whose code is not within any explanation of a one-step flip."""
    r = p["r"]
    e = int(r["expert_of_row"][row])
    c = int(r["col_of_row"][row])
    v, E = ox._gemm_rows(p["gathered"][[row]], d["gate_up_weight"][e], p["xs_layout"][:, [c]],
                         d["gate_up_weight_scale"][e])
    g, u, ge, ue = v[0, :I], v[0, I:], E[0, :I], E[0, I:]
    amb = (ox.round_sig(g - ge, 8) != ox.round_sig(g + ge, 8)) | (ox.round_sig(u - ue, 8) != ox.round_sig(u + ue, 8))
    code = p["codes"][row].view(torch.uint8).int()
    ok = ~amb & ((code & 0x7F) > 8) & ((code & 0x7F) < 0x70)
    return int(ok.nonzero()[0])


def _step(codes, row, col, n):
    out = codes.clone()
    b = out.view(torch.uint8)
    b[row, col] = int(b[row, col]) + n  # magnitude +n steps (sign bit untouched for mid-range codes)
    return out


def test_gateup_rejects_two_step_code(case):
    d, p = case
    row = int(ox.rows_to_check(p["r"], seed=1)[3])
    col = _far_element(d, p, row)
    with pytest.raises(AssertionError, match="off by 2"):
        _gateup(d, p, _step(p["codes"], row, col, 2))


def test_gateup_rejects_unexplained_flip(case):
    d, p = case
    row = int(ox.rows_to_check(p["r"], seed=1)[3])
    col = _far_element(d, p, row)
    # a one-step flip on a code far from any e4m3 boundary: the value sits mid-interval
    with pytest.raises(AssertionError, match="unexplained"):
        _gateup(d, p, _step(p["codes"], row, col, 1))


# ------------------------------------------------------------------------------------------------
# Down
# ------------------------------------------------------------------------------------------------
def _down(d, p, out, rows):
    y, B = ox.down_exact(p["codes"], p["di_layout"], p["r"], d["down_weight"],
                         d["down_weight_scale"], rows)
    return ox.check_down(out, y, B)


def test_down_passes(case):
    d, p = case
    rows = ox.rows_to_check(p["r"], seed=2)
    assert _down(d, p, p["down_out"][rows], rows) <= 1.0


def test_down_rejects_scale_from_next_n_block(case):
    d, p = case
    rows = ox.rows_to_check(p["r"], seed=2)
    dws = d["down_weight_scale"].clone()
    dws[:, 0] = dws[:, 1]
    y, _ = ox.down_exact(p["codes"], p["di_layout"], p["r"], d["down_weight"], dws, rows)
    with pytest.raises(AssertionError, match="down"):
        _down(d, p, y.to(torch.bfloat16), rows)


def test_down_rejects_k_block_scale_from_next_block(case):
    d, p = case
    rows = ox.rows_to_check(p["r"], seed=2)
    lay = p["di_layout"].clone()
    lay[0] = lay[1]
    y, _ = ox.down_exact(p["codes"], lay, p["r"], d["down_weight"], d["down_weight_scale"], rows)
    with pytest.raises(AssertionError, match="down"):
        _down(d, p, y.to(torch.bfloat16), rows)


# ------------------------------------------------------------------------------------------------
# reduce
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def shared_case():
    d = make_moe_blockwise_routed_inputs(T, K, H, I, E_TOTAL, routing="other_ranks", size_ep=4,
                                         rank_ep=1, shared=True, seed=4)
    return d, _pipeline(d)


def _reduce(d, p, out):
    o, B = ox.reduce_exact(p["down_out"], p["r"]["topk_pos"], d["topk_scale"], d["shared_output"])
    return ox.check_down(out, o, B, tag="reduce")


def test_reduce_passes(shared_case):
    d, p = shared_case
    assert _reduce(d, p, p["out"]) <= 1.0


def test_reduce_rejects_rolled_topk_scale(shared_case):
    d, p = shared_case
    o, _ = ox.reduce_exact(p["down_out"], p["r"]["topk_pos"], d["topk_scale"].roll(1, dims=1),
                           d["shared_output"])
    with pytest.raises(AssertionError, match="reduce"):
        _reduce(d, p, o.to(torch.bfloat16))


def test_reduce_rejects_dropped_shared_output(shared_case):
    d, p = shared_case
    o, _ = ox.reduce_exact(p["down_out"], p["r"]["topk_pos"], d["topk_scale"], None)
    with pytest.raises(AssertionError, match="reduce"):
        _reduce(d, p, o.to(torch.bfloat16))


# ------------------------------------------------------------------------------------------------
# guards of the checks themselves
# ------------------------------------------------------------------------------------------------
def test_gateup_rejects_unwritten_code(case):
    """A NaN code (the scratch sentinel 0x7F, one ordinal step from 448) is never a flip."""
    d, p = case
    row = int(ox.rows_to_check(p["r"], seed=1)[3])
    codes = p["codes"].clone()
    codes.view(torch.uint8)[row, 7] = 0x7F
    with pytest.raises(AssertionError, match="NaN codes"):
        _gateup(d, p, codes)


def test_accumulation_probe(case):
    """The probe is 0 on correctly rounded outputs and rejects a value rounded to the neighbouring
    bf16 where the exact value is far from the boundary (an accumulation error far beyond E)."""
    d, p = case
    rows = ox.rows_to_check(p["r"], seed=2)
    y, B = ox.down_exact(p["codes"], p["di_layout"], p["r"], d["down_weight"],
                         d["down_weight_scale"], rows)
    out = p["down_out"][rows]
    assert ox.accumulation_probe(out, y, B) <= 1.0
    r = ox.round_sig(y, 8)
    frac = ((y - r).abs() / torch.exp2(torch.floor(torch.log2(r.abs())) - 7)).flatten()
    i = int(torch.where(frac < 0.1, r.abs().flatten(), torch.zeros_like(frac)).argmax())
    bad = out.clone()
    v = float(r.flatten()[i])
    bad.view(-1)[i] = torch.tensor(v * (1 + 2.0 ** -7)).to(torch.bfloat16)  # the next bf16 up
    with pytest.raises(AssertionError, match="accumulation error"):
        ox.accumulation_probe(bad, y, B)
