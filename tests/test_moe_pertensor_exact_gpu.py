"""Per-tensor FusedMoE (hpc.fuse_moe) against the oracle on inputs with O(1) outputs, with
tolerances relative to the output RMS (see tests/test_moe_pertensor_exact_cpu.py, which shows the
check rejects swapped top-k scales, a replaced expert, an ignored activation scale and a doubled
Down scale). Covers use_bf16_mul both ways, rank_ep > 0 with experts of other ranks, shared_output,
and routing with repeated small experts. Each case prints `MOE <id> ...` (visible with -s)."""
import pytest

from test_moe_pertensor_exact_cpu import CASES, case_id, check, make, run_oracle

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_fuse_moe_pertensor_exact(hpc, c):
    d = make(c)
    use_bf16_mul = c[8]
    cu = {k: (v.cuda() if hasattr(v, "cuda") else v) for k, v in d.items()}
    my = hpc.fuse_moe(cu["x"], cu["gate_up_weight"], cu["down_weight"], cu["gate_up_scale"],
                      cu["down_scale"], cu["act_scale"], cu["topk_ids"], cu["topk_scale"],
                      d["rank_ep"], d["num_expert_total"], use_bf16_mul=use_bf16_mul,
                      shared_output=cu["shared_output"])
    ok, s = check(my, run_oracle(d, use_bf16_mul))
    print(f"MOE {case_id(c)} rms={s['rms']:.3f} outside={s['outside']} "
          f"max_err/rms={s['max_err_rms']:.4f} rel={s['rel']:.3e}")
    assert ok, s
