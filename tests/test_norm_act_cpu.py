"""Fused RMSNorm -> FP8 and the masked per-expert activation quantisers without a GPU: the oracles
against the reference's own ground truth (tests/golden/norm_*.npz, masked_act_*.npz), the operator
surface, the launchers' argument checks, and simulated kernel bugs that the GPU test's checks must
reject on that test's own cases."""
import ctypes
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import masked_act as oact
from oracle import normalization as on
from synth import act as sa
from synth import normalization as sn

G = Path(__file__).resolve().parent / "golden"
NAMES = ["fused_rmsnorm_with_scale", "masked_act_mul_and_quant", "masked_act_mul_and_blockwise_quant"]


def _bf16(a):
    return torch.from_numpy(a).view(torch.bfloat16)


def _ref_allclose(gt, my, atol=1e-8, rtol=1e-5):
    """reference tests/utils.py allclose (torch.allclose in fp32)."""
    return torch.allclose(torch.as_tensor(gt).float(), torch.as_tensor(my).float(), atol=atol, rtol=rtol)


# ---- the oracles against the reference's own functions ------------------------------------------
@pytest.mark.parametrize("H", [320, 4096, 5120])
@pytest.mark.parametrize("is_moe", [False, True])
def test_norm_oracle_matches_reference_golden(H, is_moe):
    z = np.load(G / f"norm_h{H}_{'moe' if is_moe else 'plain'}.npz")
    x, w, sc, eps = _bf16(z["x"]), _bf16(z["w"]), z["scale"], float(z["eps"][0])
    y = on.rmsnorm(x, w, eps)
    assert _ref_allclose(z["gt_fp32"], y)  # reference test_normalization.py:64
    for key, s in (("gt", sc[0]), ("gt2", sc[-1])):
        q = torch.from_numpy(on.e4m3_code(y / float(s))).view(torch.float8_e4m3fn).float()
        assert _ref_allclose(_bf16(z[key]).float(), q, atol=0.15, rtol=0.0125)  # :65-66


@pytest.mark.parametrize("tag", ["a", "b"])
def test_masked_oracle_matches_reference_golden(tag):
    z = np.load(G / f"masked_act_{tag}.npz")
    gu, sc = _bf16(z["gate_up"]), torch.from_numpy(z["scale"])
    # per-tensor: the same fp32 expression as the reference function, so every code is equal
    q = oact.masked_act_mul_and_quant(gu, sc)
    assert np.array_equal(q.view(torch.uint8).numpy(), z["gt"])
    # blockwise: the kernel multiplies by 1 / (sc + 1e-8) where the reference divides
    qb, s = oact.masked_act_mul_and_blockwise_quant(gu)
    assert np.array_equal(s.numpy(), z["gt_scale"])
    gt = torch.from_numpy(z["gt_block"]).view(torch.float8_e4m3fn).float()
    assert _ref_allclose(gt, qb.float(), atol=32, rtol=0.0125)  # reference test_act.py:168
    bad, step = oact.fp8_mismatch(qb, torch.from_numpy(z["gt_block"]))
    assert bad <= 0.001 * qb.numel() and step <= 1


# ---- surface and argument checks ------------------------------------------------------------------
def test_schemas_and_exports(hpc):
    from test_api_surface import _canon

    ref = json.loads((G / "reference_schemas.json").read_text())
    for n in NAMES:
        assert _canon(getattr(torch.ops.hpc, n).default._schema) == _canon("hpc::" + ref[n])
    for n in NAMES + ["masked_act_mul_and_quant"]:
        assert callable(getattr(hpc, n))
    import types

    assert isinstance(hpc.normalization, types.ModuleType)
    assert hpc.normalization.fused_rmsnorm_with_scale is hpc.fused_rmsnorm_with_scale


def _buf(n, align_off=0):
    b = ctypes.create_string_buffer(n + 64)
    a = ctypes.addressof(b)
    return b, ((a + 15) // 16) * 16 + align_off


def test_launchers_reject_bad_arguments(hpc):
    lib = hpc._ffi.lib
    _keep, p = _buf(1 << 16)
    _keep2, odd = _buf(1 << 16, 4)

    def norm(H, x=p, moe=0):
        return lib.hpc_fused_rmsnorm_with_scale_async(x, p, p, p, p, p, 1e-6, 4, H, moe, None)

    assert norm(12) == 1 and b"multiple of 8" in lib.hpc_last_error()
    assert norm(0) == 1 and b"multiple of 8" in lib.hpc_last_error()
    assert norm(16392) == 1 and b"16384" in lib.hpc_last_error()
    assert norm(4096, x=odd) == 1 and b"aligned" in lib.hpc_last_error()
    assert lib.hpc_fused_rmsnorm_with_scale_async(p, p, p, None, None, p, 1e-6, 4, 64, 1, None) == 1
    assert b"is_moe" in lib.hpc_last_error()

    def masked(C, N=64, T=16, x=p, blockwise=False):
        if blockwise:
            return lib.hpc_masked_act_mul_and_blockwise_quant_async(p, p, x, p, N, C, T, None)
        return lib.hpc_masked_act_mul_and_quant_async(p, x, p, p, N, C, T, None)

    assert masked(12) == 1 and b"multiple of 8" in lib.hpc_last_error()
    assert masked(64, blockwise=True) == 1 and b"multiple of 128" in lib.hpc_last_error()
    assert masked(256, N=60) == 1 and b"multiple of the tokens per expert" in lib.hpc_last_error()
    assert masked(256, N=64, T=0) == 1 and b"tokens per expert" in lib.hpc_last_error()
    assert masked(256, x=odd) == 1 and b"aligned" in lib.hpc_last_error()
    assert masked(256, x=odd, blockwise=True) == 1 and b"aligned" in lib.hpc_last_error()


def test_wrappers_reject_bad_input(hpc):
    # the op implementations check their arguments before the device, so CPU tensors reach them
    from hpc import act as ha
    from hpc import normalization as hn

    x = torch.zeros(4, 64, dtype=torch.bfloat16)
    w = torch.zeros(64, dtype=torch.bfloat16)
    s = torch.ones(2)
    with pytest.raises(RuntimeError, match="bfloat16"):
        hn._fused_rmsnorm_with_scale_impl(x.float(), w, s, 1e-6, False)
    with pytest.raises(RuntimeError, match="weight must be"):
        hn._fused_rmsnorm_with_scale_impl(x, w[:32], s, 1e-6, False)
    with pytest.raises(RuntimeError, match="at least 2"):
        hn._fused_rmsnorm_with_scale_impl(x, w, s[:1], 1e-6, True)
    with pytest.raises(RuntimeError, match="contiguous"):
        hn._fused_rmsnorm_with_scale_impl(x.t(), w, s, 1e-6, False)
    gu = torch.zeros(12, 512, dtype=torch.bfloat16)
    cnt = torch.zeros(5, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="CUDA"):
        ha._masked_act_mul_and_quant_impl(gu, torch.ones(1), cnt, None)


# ---- simulated bugs: each fails the GPU test's check on that test's own cases --------------------
def _emulate(x, w, eps, scale, bug=None):
    """The kernel's output (y32, q0, q1) emulated in fp32 numpy, with one simulated bug."""
    x = on._f64(x)
    w = on._f64(w).reshape(-1)
    H = x.shape[-1]
    if bug == "weight_dropped":
        w = np.ones_like(w)
    ss = (x * x).sum(-1, keepdims=True)
    e = float(np.float32(eps))
    m = {"mean_h_minus_1": ss / (H - 1) + e, "eps_inside_mean": (ss + e) / H}.get(bug, ss / H + e)
    r = 1 / np.sqrt(m)
    if bug == "eps_outside_rsqrt":
        r = 1 / (np.sqrt(ss / H) + e)
    if bug == "neighbour_r":
        r = np.roll(r, 1, axis=0)
    y = (x * w * r).astype(np.float32).astype(np.float64)
    sc = on._f64(scale).reshape(-1)
    inv = sc if bug == "scale_multiplied" else 1 / sc

    def q(v):
        c = on.e4m3_code(v)
        if bug == "no_saturation":
            c = np.where(np.abs(v) > 464, c | 0x7F, c)  # cvt.rn without satfinite: NaN
        return c
    return y, q(y * inv[0]), q(y * inv[1])


NORM_CASES = [(264, 17), (4096, 64), (8, 3), (16384, 3)]  # (H, T) from the GPU grid


@pytest.mark.parametrize("H,T", NORM_CASES)
def test_norm_emulated_kernel_passes(H, T):
    d = sn.make_inputs(T, H, seed=0)
    res = on.check(_emulate(d["x"], d["w"], d["eps"], d["scale"]), d["x"], d["w"], d["eps"], d["scale"], True)
    assert not on.failed(res), res


@pytest.mark.parametrize("bug", ["eps_inside_mean", "eps_outside_rsqrt", "mean_h_minus_1", "weight_dropped",
                                 "neighbour_r", "scale_multiplied", "no_saturation"])
@pytest.mark.parametrize("H,T", NORM_CASES)
def test_norm_bug_caught(bug, H, T):
    if bug == "neighbour_r" and T == 1:
        pytest.skip("one row has no neighbour")
    d = sn.make_inputs(T, H, seed=0)
    out = _emulate(d["x"], d["w"], d["eps"], d["scale"], bug)
    # the GPU test checks both is_moe outputs: fp32 within the bound, e4m3 codes up to explained flips
    assert on.failed(on.check(out, d["x"], d["w"], d["eps"], d["scale"], True)), bug


MASKED_CASES = [(8, 7, 256), (32, 336, 256), (1, 1024, 256)]  # (E, T_max, C) from the GPU grid


def _masked_emulate(d, blockwise, bug=None):
    """The kernel's buffers after a call, emulated: sentinels, then oracle rows where valid."""
    gu, cnt, T = d["gate_up"], d["num_per_expert"], d["T_max"]
    N, C = gu.shape[0], gu.shape[1] // 2
    out, osc = sa.sentinel_outputs(N, C)
    out, osc = out.view(torch.uint8).clone(), osc.clone()
    E = cnt.numel()
    keep = sa.valid_rows(cnt, T)
    if bug == "masked_row_written":
        keep = keep.clone()
        keep[int(torch.nonzero(~keep)[0])] = True
    if bug == "expert_row_mod_e":
        r = torch.arange(N)
        keep = r // E < cnt.clamp(0, T)[r % E]  # (expert, token) = (row % E, row / E)
    if blockwise:
        q, s = oact.masked_act_mul_and_blockwise_quant(
            gu, amax_cols=64 if bug == "amax_64" else 128, eps=0 if bug == "eps_dropped" else 1e-8,
            transpose_scale=bug == "scales_transposed")
        osc[keep] = s[keep]
    else:
        q = oact.masked_act_mul_and_quant(gu, d["scale"])
    out[keep] = q.view(torch.uint8)[keep]
    return out.view(torch.float8_e4m3fn), (osc if blockwise else None)


def _masked_res(d, blockwise, bug=None):
    out, osc = _masked_emulate(d, blockwise, bug)
    N, C = d["gate_up"].shape[0], d["gate_up"].shape[1] // 2
    return oact.masked_check(out, osc, d["gate_up"], d["num_per_expert"], d["T_max"],
                             sa.sentinel_outputs(N, C), scale=d["scale"])


@pytest.mark.parametrize("E,T,C", MASKED_CASES)
@pytest.mark.parametrize("blockwise", [False, True])
def test_masked_emulated_kernel_passes(E, T, C, blockwise):
    d = sa.make_inputs(E, T, C, seed=1)
    res = _masked_res(d, blockwise)
    assert oact.masked_ok(res) and res["code_bad"] == 0, res


@pytest.mark.parametrize("bug,blockwise", [("masked_row_written", False), ("masked_row_written", True),
                                           ("expert_row_mod_e", False), ("expert_row_mod_e", True),
                                           ("scales_transposed", True), ("amax_64", True),
                                           ("eps_dropped", True)])
@pytest.mark.parametrize("E,T,C", MASKED_CASES)
def test_masked_bug_caught(bug, blockwise, E, T, C):
    if bug == "expert_row_mod_e" and E == 1:
        pytest.skip("row % 1 is the right expert")
    if bug == "scales_transposed" and C == 128:
        pytest.skip("one block per row has no transpose")
    d = sa.make_inputs(E, T, C, seed=1)
    assert not oact.masked_ok(_masked_res(d, blockwise, bug)), bug
