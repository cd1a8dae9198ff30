"""The per-tensor FusedMoE check of tests/test_moe_pertensor_exact_gpu.py is not vacuous (CPU only).

Inputs from synth.moe.make_moe_pertensor_inputs give O(1) outputs. The oracle
(oracle.moe.fuse_moe_pertensor, the reference's in-test function) fed a mutated input, i.e. what
a kernel bug would compute, must fail `check`, and the unmutated oracle must pass it.
"""
import pytest
import torch

from oracle import moe as om
from synth.moe import make_moe_pertensor_inputs

# Tolerances relative to the output RMS. As for the blockwise MoE (DESIGN §5), the e4m3
# re-quantisation of the Gate-Up activation can flip one code where the kernel's fp32 summation
# order moves a bf16 Gate-Up value across a rounding point; a flip moves the Down output of that
# (token, expert) row by about half a code step times one weight column, so a few elements may
# leave the element-wise tolerance. Those are capped, and the relative L2 error is bounded.
ATOL_RMS = 0.01     # element-wise: |my - gt| <= ATOL_RMS * rms(gt) + RTOL * |gt| ...
RTOL = 0.01
OUTLIER_PPM = 50    # ... except this many elements per million, each within OUTLIER_CAP_RMS * rms
OUTLIER_CAP_RMS = 0.05
REL_L2 = 4e-3


def check(my, gt):
    """Returns (ok, stats)."""
    my, gt = my.double().cpu(), gt.double().cpu()
    rms = float(gt.pow(2).mean().sqrt())
    err = (my - gt).abs()
    finite = bool(torch.isfinite(my).all())
    bad = int((err > ATOL_RMS * rms + RTOL * gt.abs()).sum()) if finite else my.numel()
    cap = float(err.max()) / rms if finite else float("inf")
    rel = float((my - gt).norm() / gt.norm()) if finite else float("inf")
    ok = (finite and bad <= OUTLIER_PPM * 1e-6 * my.numel() and cap <= OUTLIER_CAP_RMS
          and rel <= REL_L2)
    return ok, dict(rms=rms, outside=bad, max_err_rms=cap, rel=rel)


def run_oracle(d, use_bf16_mul):
    return om.fuse_moe_pertensor(d["x"], d["gate_up_weight"], d["down_weight"], d["gate_up_scale"],
                                 d["down_scale"], d["act_scale"], d["topk_ids"], d["topk_scale"],
                                 d["rank_ep"], d["shared_output"], use_bf16_mul)


CASES = [
    # (T, K, H, I, E_total, size_ep, rank_ep, shared, use_bf16_mul, routing)
    (128, 8, 512, 512, 32, 1, 0, False, True, "uniform"),
    (128, 8, 512, 512, 32, 1, 0, False, False, "uniform"),
    (200, 8, 1024, 192, 64, 4, 2, True, True, "uniform"),
    (200, 8, 1024, 192, 64, 4, 3, True, False, "uniform"),
    (3, 8, 512, 256, 16, 1, 0, True, True, "uniform"),
    (64, 6, 512, 256, 32, 2, 1, False, True, "repeat"),
]


def case_id(c):
    return f"T{c[0]}-H{c[2]}-I{c[3]}-E{c[4]}-ep{c[6]}of{c[5]}-sh{int(c[7])}-bf16mul{int(c[8])}-{c[9]}"


def make(c):
    T, K, H, I, E_total, size_ep, rank_ep, shared, _, routing = c
    return make_moe_pertensor_inputs(T, K, H, I, E_total, size_ep, rank_ep, shared, routing,
                                     seed=T + H)


def mutations(d):
    E = d["gate_up_weight"].shape[0]
    local = d["topk_ids"].long() - d["rank_ep"] * E
    local = local[(local >= 0) & (local < E)]
    busy = int(torch.bincount(local, minlength=E).argmax())  # the most used local expert
    g = torch.Generator().manual_seed(5)
    out = {}
    # scales read from the neighbouring top-k slot (every slot moves: with sorted ids and a high
    # rank_ep only the last slots hold this rank's experts)
    out["topk_scale_slots_shifted"] = dict(d, topk_scale=d["topk_scale"].roll(1, dims=1).contiguous())
    guw = d["gate_up_weight"].clone()
    guw[busy] = torch.randn(guw[busy].shape, generator=g).to(torch.float8_e4m3fn)
    out["expert_gate_up_replaced"] = dict(d, gate_up_weight=guw)
    out["act_scale_ignored"] = dict(d, act_scale=torch.ones_like(d["act_scale"]))
    ds = d["down_scale"].clone()
    ds[busy] *= 2
    out["expert_down_scale_x2"] = dict(d, down_scale=ds)
    return out


@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_moe_pertensor_check_discriminates(c):
    d = make(c)
    gt = run_oracle(d, c[8])
    assert 0.2 < check(gt, gt)[1]["rms"] < 5, "outputs are not O(1)"
    assert check(gt, gt)[0]
    if c[8]:  # the other activation product rounding stays inside the tolerance's scale
        assert check(run_oracle(d, False), gt)[1]["rel"] < 10 * REL_L2
    undetected = [(n, s) for n, m in mutations(d).items()
                  for ok, s in [check(run_oracle(m, c[8]), gt)] if ok]
    assert not undetected, undetected
