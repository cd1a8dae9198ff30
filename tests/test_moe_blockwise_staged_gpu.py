"""The blockwise FusedMoE pipeline checked stage by stage against oracle/moe_exact.py.

Every scratch buffer is filled with a sentinel first (NaN for f32 / bf16, 0x7F = e4m3 NaN for fp8,
-7 for ints), so a stage that leaves an element it owns unwritten, or reads one it should not,
shows up whatever the allocator handed out. The grid runs scale granules 8, 16, 32 and 48 (and the
65-96 / 97-128 / 129-144 buckets, which map back to 48 / 32 / 48; granule 64 is what
test_moe_gpu.py's blockwise grid runs) with a partial Down N tile, kpad4 != K/128 on both GEMMs,
hot, sparse and other-rank routings, the C3 shape and the 512-expert limit."""
import pytest
import torch

from oracle import moe_exact as ox
from synth.moe import make_moe_blockwise_routed_inputs

pytestmark = pytest.mark.gpu

SENTINEL = {torch.float32: float("nan"), torch.bfloat16: float("nan"), torch.int32: -7}


def _fill(s):
    for t in s.values():
        if not isinstance(t, torch.Tensor):
            continue
        if t.dtype == torch.float8_e4m3fn:
            t.view(torch.uint8).fill_(0x7F)
        else:
            t.fill_(SENTINEL[t.dtype])


def _run_staged(hpc, d):
    from hpc.fuse_moe import _blockwise_scratch, _launch_blockwise

    c = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in d.items()}
    s = _blockwise_scratch(c["x"], c["gate_up_weight"], c["topk_ids"], c["num_expert_total"])
    _fill(s)
    y = torch.full((c["x"].size(0), c["x"].size(1)), float("nan"), dtype=torch.bfloat16,
                   device="cuda")
    args = (c["x"], c["x_scale"], c["gate_up_weight"], c["gate_up_weight_scale"],
            c["down_weight"], c["down_weight_scale"], c["topk_ids"], c["topk_scale"],
            c["shared_output"], c["rank_ep"], c["num_expert_total"])
    _launch_blockwise(y, *args, s)
    public = hpc.fuse_moe_blockwise(*args[:8], c["rank_ep"], c["num_expert_total"],
                                    c["shared_output"])
    torch.cuda.synchronize()
    assert torch.equal(public.view(torch.int16), y.view(torch.int16)), \
        "public op differs from the staged launch"
    return y.cpu(), {k: (v.cpu() if isinstance(v, torch.Tensor) else v) for k, v in s.items()}


def _check_all(hpc, d, tag, seed=0):
    y, s = _run_staged(hpc, d)
    E = d["gate_up_weight"].size(0)
    r = ox.route(d["topk_ids"], E, d["rank_ep"], d["num_expert_total"])
    ox.check_route(r, d["x"], d["x_scale"], s)
    rows = ox.rows_to_check(r, seed=seed)
    st = dict(tag=tag, granule=r["granule"], rows=int(r["src_token"].numel()),
              checked=int(rows.numel()), flips=0, explained=0, down=0.0, reduce=0.0,
              down_acc=0.0, reduce_acc=0.0)
    if rows.numel():
        g = ox.check_gateup(s["gate_up_input"], s["gate_up_input_scale"], r, d["gate_up_weight"],
                            d["gate_up_weight_scale"], rows, s["down_input"], s["down_input_scale"])
        st.update(flips=g["flips"], explained=g["explained"])
        yd, B = ox.down_exact(s["down_input"], s["down_input_scale"], r, d["down_weight"],
                              d["down_weight_scale"], rows)
        st["down"] = ox.check_down(s["down_output"][rows], yd, B, tag=f"{tag} down")
        st["down_acc"] = ox.accumulation_probe(s["down_output"][rows], yd, B, tag=f"{tag} down")
    o, B = ox.reduce_exact(s["down_output"], s["topk_pos"], d["topk_scale"], d["shared_output"])
    st["reduce"] = ox.check_down(y, o, B, tag=f"{tag} reduce")
    st["reduce_acc"] = ox.accumulation_probe(y, o, B, tag=f"{tag} reduce")
    print(f"\n[{tag}] granule {st['granule']} rows {st['rows']} checked {st['checked']} "
          f"flips {st['flips']} (explained {st['explained']}) down err/B {st['down']:.3f} "
          f"acc/E>={st['down_acc']:.3f} reduce err/B {st['reduce']:.3f} "
          f"acc/E>={st['reduce_acc']:.3f}")
    return st


GRID_T = [200, 400, 700, 1400, 2000, 2250]  # granules 16, 32, 48, 48 (65-96), 32 (97-128), 48 (129-144)
SHAPES = [(640, 384), (1152, 256)]


@pytest.mark.parametrize("H,I", SHAPES)
def test_staged_sparse_decode(hpc, H, I):
    """T = 16 over 128 experts: avg 1 -> granule 8, most experts empty."""
    d = make_moe_blockwise_routed_inputs(16, 8, H, I, 128, routing="sparse", seed=7)
    st = _check_all(hpc, d, f"T16 sparse H{H} I{I}")
    assert st["granule"] == 8


@pytest.mark.parametrize("H,I", SHAPES)
@pytest.mark.parametrize("T", GRID_T)
@pytest.mark.parametrize("routing", ["uniform", "hot", "other_ranks"])
def test_staged_grid(hpc, T, H, I, routing):
    kw = dict(size_ep=4, rank_ep=1, shared=True) if routing == "other_ranks" else {}
    d = make_moe_blockwise_routed_inputs(T, 8, H, I, 128, routing=routing, seed=T + H, **kw)
    st = _check_all(hpc, d, f"T{T} {routing} H{H} I{I}", seed=T)
    assert st["granule"] == ox.scale_granule(T * 8 // 128)


def test_staged_c3_shape(hpc):
    """H 4096, I 14336, 8 local experts of 128 (size_ep 16), T = 512: the K = 14336 Down GEMM with
    the fused scale layout."""
    d = make_moe_blockwise_routed_inputs(512, 8, 4096, 14336, 128, routing="other_ranks",
                                         size_ep=16, rank_ep=3, seed=12)
    _check_all(hpc, d, "C3 shape T512 ep16")


def test_staged_512_local_experts(hpc):
    d = make_moe_blockwise_routed_inputs(256, 8, 256, 256, 512, routing="uniform", seed=13)
    _check_all(hpc, d, "512 experts")


def test_513_local_experts_rejected(hpc):
    d = make_moe_blockwise_routed_inputs(16, 8, 256, 256, 513, routing="uniform", seed=14)
    c = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in d.items()}
    with pytest.raises(RuntimeError, match="local experts 513 not in"):
        hpc.fuse_moe_blockwise(c["x"], c["x_scale"], c["gate_up_weight"], c["gate_up_weight_scale"],
                               c["down_weight"], c["down_weight_scale"], c["topk_ids"],
                               c["topk_scale"], 0, 513)
