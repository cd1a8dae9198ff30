"""ORACLE — test infrastructure only (never imported by the product).

Masked per-expert activation quantisers (hpc.masked_act_mul_and_quant,
hpc.masked_act_mul_and_blockwise_quant; reference tests/test_act.py `ref_masked_act_mul_and_quant`,
`ref_masked_act_mul_and_blockwise_quant`), computed the kernel's way in fp32: v = silu(g) * u, then
e4m3(v * scale[0]), or per 128 columns sc = amax / 448 and e4m3(v * (1 / (sc + 1e-8))) (a multiply
by the reciprocal, where the reference test divides). Pinned by tests/golden/masked_act_*.npz.
"""
import torch


def _silu_mul(gate_up):
    gate, up = torch.chunk(gate_up.float(), 2, dim=-1)
    return gate / (1 + (-gate).exp()) * up


def _e4m3(v):
    return v.clamp(-448.0, 448.0).to(torch.float8_e4m3fn)


def masked_act_mul_and_quant(gate_up, scale):
    """Every row of the padded layout (validity is the check's business): e4m3(silu(g) * u * s)."""
    return _e4m3(_silu_mul(gate_up) * scale.float().reshape(-1)[0])


def masked_act_mul_and_blockwise_quant(gate_up, amax_cols=128, eps=1e-8, transpose_scale=False):
    """(e4m3 [N, C], sc f32 [N, C / 128]) of every row. `amax_cols` and `eps` exist for the
    simulated-bug tests (an amax over 64 columns, the +1e-8 dropped)."""
    v = _silu_mul(gate_up)
    n, c = v.shape
    amax = v.abs().reshape(n, -1, amax_cols).amax(-1)
    sc = amax / 448.0
    inv = 1.0 / (sc + eps) if eps else 1.0 / sc
    q = _e4m3(v * inv.repeat_interleave(amax_cols, -1))
    sc = sc.reshape(n, -1, 128 // amax_cols)[..., 0].contiguous()
    if transpose_scale:
        sc = sc.t().contiguous().reshape(n, -1)
    return q, sc


def fp8_mismatch(my, gt):
    """(#codes that differ, max |difference| in e4m3 code steps) of two e4m3 / uint8 tensors."""
    a = my.contiguous().view(torch.uint8).cpu().to(torch.int32)
    b = gt.contiguous().view(torch.uint8).cpu().to(torch.int32)
    diff = a != b
    step = ((a & 0x7F) - (b & 0x7F)).abs()[diff]
    return int(diff.sum()), int(step.max()) if step.numel() else 0


SCALE_REL = 2.0 ** -20


def masked_check(out, out_scale, gate_up, num_per_expert, T_max, sentinels, scale=None):
    """The GPU test's check of one masked call. `out` / `out_scale` (None for per-tensor) are the
    kernel's buffers, which held `sentinels` = (out0, scale0) before the call. Returns a dict:
    invalid rows changed (must be 0), code and scale mismatches on valid rows with the largest code
    step, and the number of valid elements (the 20 ppm flip allowance is taken of it)."""
    from synth.act import valid_rows

    keep = valid_rows(num_per_expert.cpu(), T_max)
    o = out.contiguous().view(torch.uint8).cpu()
    o0 = sentinels[0].contiguous().view(torch.uint8).cpu()
    res = {"invalid_changed": int((o[~keep] != o0[~keep]).sum())}
    if out_scale is None:
        gt = masked_act_mul_and_quant(gate_up.cpu(), scale.cpu())
    else:
        gt, gs = masked_act_mul_and_blockwise_quant(gate_up.cpu())
        s = out_scale.contiguous().view(torch.int32).cpu()
        s0 = sentinels[1].contiguous().view(torch.int32).cpu()
        res["invalid_changed"] += int((s[~keep] != s0[~keep]).sum())
        # CUDA expf is within 2 ulp of the CPU's, so silu(g) * u and with it amax / 448 may differ
        # by a few ulp: scales must agree to 2^-20 relative (16 ulp), sentinels (NaN) never do
        sv, gv = s[keep].view(torch.float32), gs[keep]
        res["scale_bad"] = int((~((sv - gv).abs() <= SCALE_REL * gv.abs())).sum())
    res["code_bad"], res["step"] = fp8_mismatch(o[keep], gt.view(torch.uint8)[keep])
    res["valid"] = int(keep.sum()) * o.shape[1]
    return res


def masked_ok(res):
    """The GPU test's acceptance: invalid rows untouched; codes exact on valid rows except for
    <= 20 ppm one-code flips from CUDA expf's <= 2 ulp (as test_act_gpu.py allows); every scale
    within SCALE_REL of the oracle's."""
    allow = max(2, 20e-6 * res["valid"])
    return (res["invalid_changed"] == 0 and res["code_bad"] <= allow and res["step"] <= 1
            and res.get("scale_bad", 0) == 0)
