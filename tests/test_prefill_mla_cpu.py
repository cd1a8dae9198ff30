"""CPU side of the MLA prefill: the exact oracle against brute force, its mutants, the C launcher's
rejections and the fake op."""
import ctypes
import math

import pytest
import torch

from oracle import prefill_mla as om
from synth import prefill_mla as sm

CASES = [
    # (q_lens, kv_lens, H, kind)
    ([1, 130, 0, 40], [1, 200, 5, 40], 4, "random"),
    ([129, 7, 60], [129, 70, 30], 2, "pe"),
    ([3, 131, 20], [64, 131, 150], 3, "edge"),
    ([50, 127], [177, 127], 1, "edge"),
]


@pytest.fixture(scope="module")
def cases():
    return [sm.make_case(ql, kl, h, seed=i, kind=k) for i, (ql, kl, h, k) in enumerate(CASES)]


def _brute(d):
    """Row by row, head by head, from the definition: fp64, no batching, no bound."""
    q, kn, kp, v = (d[k].double() for k in ("q", "k_nope", "k_pe", "v"))
    y = torch.full((q.shape[0], q.shape[1], 128), math.nan, dtype=torch.float64)
    cq, ck = d["cu_seqlens_q"].tolist(), d["cu_seqlens_kv"].tolist()
    for b in range(len(cq) - 1):
        nq, nk = cq[b + 1] - cq[b], ck[b + 1] - ck[b]
        for i in range(nq):
            n_vis = max(0, min(nk, nk - nq + i + 1))
            for h in range(q.shape[1]):
                if n_vis == 0:
                    y[cq[b] + i, h] = 0
                    continue
                keys = torch.cat([kn[ck[b]:ck[b] + n_vis, h], kp[ck[b]:ck[b] + n_vis]], 1)
                s = keys @ q[cq[b] + i, h] * d["scale"]
                y[cq[b] + i, h] = torch.softmax(s, 0) @ v[ck[b]:ck[b] + n_vis, h]
    return y


def test_exact_matches_brute_force(cases):
    for d in cases:
        exact, bound = om.mla_prefill_exact(d["q"], d["k_nope"], d["k_pe"], d["v"],
                                            d["cu_seqlens_q"], d["cu_seqlens_kv"], d["scale"])
        ref = _brute(d)
        assert torch.equal(torch.isnan(exact), torch.isnan(ref))
        ok = ~torch.isnan(ref)
        assert torch.allclose(exact[ok], ref[ok], rtol=1e-10, atol=1e-10)
        assert (bound[ok] >= 0).all() and torch.isfinite(bound[ok]).all()


def test_rows_subset_matches_full(cases):
    d = cases[0]
    a = (d["q"], d["k_nope"], d["k_pe"], d["v"], d["cu_seqlens_q"], d["cu_seqlens_kv"], d["scale"])
    full, fb = om.mla_prefill_exact(*a)
    rows = torch.zeros(d["q"].shape[0], dtype=torch.bool)
    rows[::7] = True
    part, pb = om.mla_prefill_exact(*a, rows=rows)
    assert torch.equal(part[rows], full[rows]) and torch.equal(pb[rows], fb[rows])
    assert torch.isnan(part[~rows]).all()


def test_no_visible_key_rows_are_zero(cases):
    d = cases[2]
    small = sm.make_case([10], [4], 2, seed=9)  # 10 queries over 4 keys: rows 0-5 see none
    y, b = om.mla_prefill_exact(small["q"], small["k_nope"], small["k_pe"], small["v"],
                                small["cu_seqlens_q"], small["cu_seqlens_kv"], small["scale"])
    assert (y[:6] == 0).all() and (b[:6] == 0).all() and (y[6:].abs().sum(-1) > 0).all()
    assert torch.isnan(d["latent"][:, :512]).all() and torch.isnan(d["kv"][-sm.SLACK:]).all()


def test_lossy_oracle_passes_exact_check(cases):
    for d in cases:
        r = om.check(om.mla_prefill_exact(d["q"], d["k_nope"], d["k_pe"], d["v"], d["cu_seqlens_q"],
                                          d["cu_seqlens_kv"], d["scale"], lossy=True)[0], d)
        assert r["ok_a"] and r["ok_b"], (d["kind"], r)


@pytest.mark.parametrize("mutation", om.MUTATIONS)
def test_every_mutation_is_caught(cases, mutation):
    caught, applicable = [], []
    for i, d in enumerate(cases):
        if not sm.applicable(d, mutation):
            continue
        applicable.append(i)
        r = om.check(om.mutant(d, mutation), d)
        if not (r["ok_a"] and r["ok_b"]):
            caught.append(i)
    print(f"mutation {mutation}: caught by cases {caught} of {applicable}")
    assert applicable, f"no case exercises {mutation}"
    assert caught, mutation


def test_launcher_rejections(hpc):
    lib = hpc._ffi.lib
    P = ctypes.c_void_p(1 << 20)
    I = ctypes.cast(P, ctypes.POINTER(ctypes.c_int))

    def call(**kw):
        a = dict(ptr_q=P, num_batch=2, total_q=300, total_kv=400, max_q=200, heads=16, dqk=192,
                 dv=128, ldY=16 * 128, ldQ=16 * 192, kn_tok=16 * 256, kn_head=256, pe_tok=576,
                 v_tok=16 * 256, v_head=256, scale=0.1)
        a.update(kw)
        return lib.hpc_attention_prefill_mla_bf16_async(
            P, a["ptr_q"], P, P, P, I, I, a["num_batch"], a["total_q"], a["total_kv"], a["max_q"],
            a["heads"], a["dqk"], a["dv"], a["ldY"], a["ldQ"], a["kn_tok"], a["kn_head"],
            a["pe_tok"], a["v_tok"], a["v_head"], a["scale"], None)

    for bad in (dict(dqk=128), dict(dqk=576), dict(dv=192), dict(heads=0), dict(heads=129),
                dict(num_batch=0), dict(total_kv=0), dict(total_q=-1), dict(scale=0.0),
                dict(scale=-1.0), dict(scale=math.inf), dict(scale=math.nan),
                dict(ptr_q=ctypes.c_void_p((1 << 20) + 8)), dict(ldQ=16 * 192 + 4),
                dict(ldQ=15 * 192), dict(ldY=16 * 128 - 8), dict(kn_tok=16 * 256 + 2),
                dict(kn_head=260), dict(pe_tok=580), dict(v_tok=0), dict(v_head=130),
                dict(max_q=1 << 30, heads=128, num_batch=1000)):
        assert call(**bad) == 1, bad
        assert lib.hpc_last_error()


def test_host_rejections(hpc):
    """The op's host side checks dtypes and shapes before devices, so each rejection shows on CPU
    tensors with its own message; a well-formed CPU call fails only on the device check."""
    from hpc.attention import _attention_prefill_mla_bf16_impl as f
    d = sm.make_case([5, 3], [9, 3], 2, seed=1)
    a = dict(q=d["q"], k_nope=d["k_nope"], k_pe=d["k_pe"], v=d["v"], cu_seqlens_q=d["cu_seqlens_q"],
             cu_seqlens_kv=d["cu_seqlens_kv"])

    def call(**kw):
        x = dict(a)
        x.update(kw)
        return f(x["q"], x["k_nope"], x["k_pe"], x["v"], x["cu_seqlens_q"], x["cu_seqlens_kv"], 5,
                 d["scale"])

    kv3 = torch.zeros(20, 3, 256, dtype=torch.bfloat16)
    bad = [
        (dict(q=d["q"].float()), "q must be bfloat16"),
        (dict(k_pe=d["k_pe"].half()), "k_pe must be bfloat16"),
        (dict(cu_seqlens_q=d["cu_seqlens_q"].long()), "cu_seqlens_q must be contiguous int32"),
        (dict(cu_seqlens_kv=d["cu_seqlens_kv"][:2]), "num_batch"),
        (dict(cu_seqlens_q=d["cu_seqlens_q"][:1], cu_seqlens_kv=d["cu_seqlens_kv"][:1]), "num_batch"),
        (dict(q=d["q"][..., :128]), "q must be"),
        (dict(q=torch.zeros(8, 129, 192, dtype=torch.bfloat16)), "num heads"),
        (dict(q=torch.zeros(8, 2, 384, dtype=torch.bfloat16)[..., :192]), "contiguous in"),
        (dict(k_nope=kv3[..., :128]), "k_nope must be"),
        (dict(v=torch.zeros(20, 2, 192, dtype=torch.bfloat16)), "v must be"),
        (dict(k_pe=torch.zeros(20, 576, dtype=torch.bfloat16)[:, 448:]), "k_pe must be"),
        (dict(k_pe=d["k_pe"][:-1]), "same total_kv"),
        (dict(v=torch.zeros(d["v"].size(0), 2, 256, dtype=torch.bfloat16)[..., ::2]),
         "rows must be contiguous"),
    ]
    for kw, msg in bad:
        with pytest.raises(RuntimeError, match=msg):
            call(**kw)
    with pytest.raises(RuntimeError, match="cuda tensor"):
        call()


def test_fake_shape(hpc):
    from torch._subclasses.fake_tensor import FakeTensorMode
    with FakeTensorMode():
        q = torch.empty(300, 16, 192, dtype=torch.bfloat16, device="cuda")
        kv = torch.empty(500, 16, 256, dtype=torch.bfloat16, device="cuda")
        lat = torch.empty(500, 576, dtype=torch.bfloat16, device="cuda")
        cu = torch.empty(3, dtype=torch.int32, device="cuda")
        y = torch.ops.hpc.attention_prefill_mla_bf16(q, kv[..., :128], lat[:, 512:], kv[..., 128:],
                                                     cu, cu, 200, 0.1, None)
        assert y.shape == (300, 16, 128) and y.dtype == torch.bfloat16 and y.device.type == "cuda"
        out = torch.empty(300, 16, 128, dtype=torch.bfloat16, device="cuda")
        assert torch.ops.hpc.attention_prefill_mla_bf16(q, kv[..., :128], lat[:, 512:],
                                                        kv[..., 128:], cu, cu, 200, 0.1,
                                                        out) is out
    assert hasattr(hpc, "attention_prefill_mla_bf16")
