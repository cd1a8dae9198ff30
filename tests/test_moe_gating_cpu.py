"""MoE top-k gating without a GPU: the fp64 oracle against the independent fp32 torch chain on the
GPU test's own cases, simulated kernel bugs that the GPU test's check must reject, the fake
registration, and the argument checks of the launcher and the Python wrapper."""
import ctypes
import importlib

import numpy as np
import pytest
import torch

from oracle import moe_gating as og
from synth import moe_gating as sg

CASES = [(name, dt, kind) for name in sg.CONFIGS for dt in ("fp32", "bf16")
         for kind in ("random", "ties")]


def _case(name, dt, kind, T=128):
    cfg = sg.CONFIGS[name]
    dtype = torch.float32 if dt == "fp32" else torch.bfloat16
    return sg.make_case(cfg, T, dtype, seed=sg.seed_of(name, dt, kind, T), kind=kind, pad=8)


def _exact_tie_rows(ref, k):
    """Rows with two equal keys among the first k + 1 of the order: torch.topk may order such a
    pair either way, the contract puts the lower id first."""
    keys = np.take_along_axis(ref["keys"], ref["order"][:, :k + 1], -1)
    return (keys[:, 1:] == keys[:, :-1]).any(-1)


@pytest.mark.parametrize("name", list(sg.CONFIGS))
@pytest.mark.parametrize("dt", ["fp32", "bf16"])
def test_oracle_matches_torch_chain(name, dt):
    c = _case(name, dt, "random")
    cfg = c["cfg"]
    ref = sg.oracle(c["x"], cfg, c["bias"])
    ids, w = sg.torch_chain(c["logits"], **sg.hpc_kwargs(cfg, c["bias"]))
    rows = ~_exact_tie_rows(ref, cfg["topk"])
    assert rows.sum() >= 32
    assert np.array_equal(ids.numpy()[rows], ref["ids"][rows])
    assert (np.abs(w.double().numpy() - ref["weights"]) <= ref["w_bound"]).all()


def test_margins_and_planted_ties_hold():
    for name, dt, kind in CASES:
        c = _case(name, dt, kind)
        ref = sg.oracle(c["x"], c["cfg"], c["bias"])
        assert og.boundary_ok(ref, c["cfg"]["topk"], c["cfg"]["topk_group"]).all()
        if kind == "ties":
            assert len(c["planted"]) >= 100, (name, dt)
            for t, lo, hi, what in c["planted"]:
                if what == "expert":
                    assert lo in ref["ids"][t] and hi not in ref["ids"][t]


# ---- simulated bugs: each fails the GPU test's check on that test's own cases --------------------
def _emulate(x, cfg, bias, bug=None):
    """The kernel's (ids, weights) emulated in fp64 with one simulated bug."""
    T, E = x.shape
    k, G, tg, f = cfg["topk"], cfg["G"], cfg["topk_group"], cfg["factor"]
    b = np.zeros(E) if bias is None else bias.double().numpy()
    if cfg["scoring"] == 0:
        e = np.exp(x - x.max(-1, keepdims=True))
        s = e / e.sum(-1, keepdims=True)
    else:
        s = 1 / (1 + np.exp(-x))
    keys = x if cfg["scoring"] == 0 and bias is None else s + b
    idx = np.broadcast_to(np.arange(E), (T, E))
    tie = -idx if bug == "ties_to_higher_id" else idx
    elig = np.ones((T, E), bool)
    if G > 1:
        gs = E // G
        member = (idx + (1 if bug == "group_boundary_off_by_one" else 0)) // gs % G
        gk = np.stack([np.where(member == g, keys, -np.inf) for g in range(G)], 1)
        top2 = -np.sort(-gk, -1)[..., :2]
        gscore = top2[..., 0] if bias is None or bug == "group_max_for_top2_sum" else top2.sum(-1)
        gorder = np.lexsort((np.broadcast_to(np.arange(G), (T, G)), -gscore), axis=-1)[:, :tg]
        if bug == "groups_chosen_by_id":
            gorder = np.broadcast_to(np.arange(tg), (T, tg))
        elig = (member[:, :, None] == gorder[:, None, :]).any(-1)
    order = np.lexsort((tie, -keys, ~elig), axis=-1)
    ids = order[:, :k]
    w = np.take_along_axis(keys if bug == "bias_in_weights" else s, ids, -1)
    if bug == "softmax_over_chosen_k":
        xe = np.exp(np.take_along_axis(x, ids, -1))
        w = xe / xe.sum(-1, keepdims=True)
    if bug == "scaling_before_renormalize":
        w = w * f
    if cfg["renormalize"] and bug != "renormalize_skipped":
        w = w / w.sum(-1, keepdims=True)
    if bug != "scaling_before_renormalize":
        w = w * f
    return ids.astype(np.int32), w


# bug -> the families whose configuration exercises it
BUGS = {
    "ties_to_higher_id": list(sg.CONFIGS),
    "group_max_for_top2_sum": ["deepseek_v3"],
    "bias_in_weights": ["deepseek_v3", "kimi_k2"],
    "renormalize_skipped": ["mixtral", "qwen3", "deepseek_v3", "kimi_k2", "qwen3_next"],
    "scaling_before_renormalize": ["deepseek_v3", "kimi_k2"],
    "groups_chosen_by_id": ["deepseek_v2", "deepseek_v3"],
    "group_boundary_off_by_one": ["deepseek_v2", "deepseek_v3"],
    "softmax_over_chosen_k": ["deepseek_v2"],
}


@pytest.mark.parametrize("name,dt,kind", CASES)
def test_emulated_kernel_passes(name, dt, kind):
    c = _case(name, dt, kind)
    ref = sg.oracle(c["x"], c["cfg"], c["bias"])
    assert not og.failed(og.check(*_emulate(c["x"], c["cfg"], c["bias"]), ref))


@pytest.mark.parametrize("bug,name", [(b, n) for b, ns in BUGS.items() for n in ns])
@pytest.mark.parametrize("dt", ["fp32", "bf16"])
def test_bug_caught(bug, name, dt):
    # the GPU test checks the random and the tie case of every family
    caught = False
    for kind in ("random", "ties"):
        c = _case(name, dt, kind)
        ref = sg.oracle(c["x"], c["cfg"], c["bias"])
        caught |= og.failed(og.check(*_emulate(c["x"], c["cfg"], c["bias"], bug), ref))
    assert caught, (bug, name, dt)


# ---- surface, fake registration, argument checks ----------------------------------------------
def test_exports_and_fake_shapes(hpc):
    from torch._subclasses.fake_tensor import FakeTensorMode

    assert hpc.GatingScore.SOFTMAX == 0 and hpc.GatingScore.SIGMOID == 1
    assert hpc.moe_topk_gating is importlib.import_module("hpc.fuse_moe").moe_topk_gating
    with FakeTensorMode():
        x = torch.empty(7, 192, device="cuda")
        ids, w = hpc.moe_topk_gating(x[:, :160], 6, num_expert_group=8, topk_group=3)
        assert ids.shape == (7, 6) and ids.dtype == torch.int32
        assert w.shape == (7, 6) and w.dtype == torch.float32
        out = (torch.empty(7, 6, dtype=torch.int32, device="cuda"),
               torch.empty(7, 6, device="cuda"))
        r = hpc.moe_topk_gating(x[:, :160], 6, topk_ids=out[0], topk_weights=out[1])
        assert r[0].shape == (7, 6) and r[1].dtype == torch.float32


def _buf(n, align_off=0):
    b = ctypes.create_string_buffer(n + 64)
    return b, ((ctypes.addressof(b) + 15) // 16) * 16 + align_off


def test_launcher_rejects_bad_arguments(hpc):
    lib = hpc._ffi.lib
    _keep, p = _buf(1 << 16)

    def call(T=4, E=256, dtype=0, k=8, scoring=1, G=8, tg=4, stride=256, bias=p, x=p):
        return lib.hpc_moe_topk_gating_async(x, bias, p, p, T, E, dtype, k, scoring, 1, G, tg,
                                             stride, 1.0, None)

    for kw, msg in ((dict(T=-1), b"negative"), (dict(E=0, G=1, tg=1), b"experts 0"),
                    (dict(E=520, G=1, tg=1, stride=520), b"[1, 512]"), (dict(k=0), b"topk 0"),
                    (dict(k=17), b"topk 17"), (dict(E=8, k=9, G=1, tg=1), b"topk 9"),
                    (dict(dtype=2), b"dtype"), (dict(scoring=2), b"scoring"),
                    (dict(G=7), b"num_expert_group 7"), (dict(G=0), b"num_expert_group 0"),
                    (dict(tg=9), b"topk_group 9"), (dict(tg=0), b"topk_group 0"),
                    (dict(G=64, tg=1), b"exceeds"), (dict(G=256, tg=8, k=8), b"at least 2"),
                    (dict(stride=200), b"row stride"), (dict(stride=258), b"row stride"),
                    (dict(x=p + 4), b"aligned"), (dict(x=None), b"null")):
        assert call(**kw) == 1, kw
        assert msg in lib.hpc_last_error(), (kw, lib.hpc_last_error())
    # T = 0 is accepted without a launch; a single row's stride is never used
    assert call(T=0) == 0
    assert call(T=0, x=None) == 0


def test_wrapper_rejects_bad_input(hpc):
    # the wrapper checks its arguments before the device, so CPU tensors reach the checks
    fm = importlib.import_module("hpc.fuse_moe")
    x = torch.zeros(4, 256)
    args = dict(topk=8, scoring=1, renormalize=True, correction_bias=torch.zeros(256),
                num_expert_group=8, topk_group=4, routed_scaling_factor=1.0, topk_ids=None,
                topk_weights=None)

    def bad(match, xx=x, **kw):
        with pytest.raises(RuntimeError, match=match):
            fm._moe_topk_gating_impl(xx, **{**args, **kw})

    bad("float32 or bfloat16", xx=x.half())
    bad("2-D", xx=x[0])
    bad("contiguous", xx=torch.zeros(256, 4).t())
    bad("outside", xx=torch.zeros(4, 520), correction_bias=None, num_expert_group=1, topk_group=1)
    bad("topk 17", topk=17)
    bad("divide", num_expert_group=3)
    bad("topk_group 9", topk_group=9)
    bad("row stride", xx=torch.zeros(4, 258)[:, :256])
    bad("correction_bias", correction_bias=torch.zeros(255))
    bad("at least 2", num_expert_group=256, topk_group=8)
    bad("topk_ids", topk_ids=torch.zeros(4, 8, dtype=torch.int64))
    bad("topk_weights", topk_weights=torch.zeros(4, 7))
    bad("CUDA")
