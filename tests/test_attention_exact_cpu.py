"""The exact-reference checks are not vacuous (CPU only).

For every input family of synth/attention_exact.py, the lossy oracle (oracle/attention.py,
oracle/prefill.py: the reference's in-test functions) passes both checks of
oracle/attention_exact.grade against the fp64 reference, and the same oracle fed a mutated input
(a wrong Q, scale, page, mask or causal limit, i.e. what a kernel bug would compute) fails one
of them.
"""
import pytest
import torch

from oracle import attention as oa
from oracle import attention_exact as ox
from oracle import prefill as op
from synth.attention_exact import make_decode_exact_inputs, make_prefill_exact_inputs

PAGE = 64


# ------------------------------------------------------------------------------------------------
# decode
# ------------------------------------------------------------------------------------------------
def _kpt_views(d):
    kv = d["kvcache"]
    d.update(kcache=kv[:, 0, :PAGE], vcache=kv[:, 1, :PAGE], k_scale=kv[:, 0, PAGE:])
    return d


def decode_lossy(d, sq, kpt):
    if kpt:
        return oa.decode_fp8_kpertoken(d["q"], d["kcache"], d["vcache"], d["block_ids"],
                                       d["kv_lens_total"], d["q_scale"], d["k_scale"],
                                       d["v_scale"], sq)
    return oa.decode_fp8_kvpertensor(d["q"], d["kvcache"][:, 0], d["kvcache"][:, 1],
                                     d["block_ids"], d["kv_lens_total"], d["q_scale"],
                                     d["k_scale"], d["v_scale"], sq)


def decode_exact(d, sq, kpt):
    k = d["kcache"] if kpt else d["kvcache"][:, 0]
    v = d["vcache"] if kpt else d["kvcache"][:, 1]
    return ox.decode_fp8_exact(d["q"], k, v, d["block_ids"], d["kv_lens_total"], d["q_scale"],
                               d["k_scale"], d["v_scale"], sq, k_per_token=kpt)


def _scale_rows_f32(kv):
    # the k-per-token scale rows of a [blocks, 2, bs + 2, Hkv, D] cache as f32 [blocks, 2, Hkv, 32]
    return kv[:, 0, PAGE:].contiguous().view(torch.float32)


def decode_mutations(d, sq, kpt):
    """name -> mutated copy of the inputs."""
    out = {}
    gen = torch.Generator().manual_seed(99)

    def cp(**kw):
        e = dict(d)
        e.update(kw)
        return _kpt_views(e) if kpt else e

    qf = d["q"].float()
    out["unrelated_q"] = cp(q=(torch.randn(qf.shape, generator=gen) * qf.std()).clamp(-440, 440)
                          .to(torch.float8_e4m3fn))  # finite codes: the scores must reject it
    out["zero_q"] = cp(q=torch.zeros_like(qf).to(torch.float8_e4m3fn))
    out["reversed_q_heads"] = cp(q=d["q"].flip(1), q_scale=d["q_scale"].flip(1))
    kv = d["kvcache"].clone()
    if kpt:
        rows = _scale_rows_f32(kv) * 2
        kv[:, 0, PAGE:] = rows.view(torch.float8_e4m3fn).reshape(kv[:, 0, PAGE:].shape)
        out["k_scale_x2"] = cp(kvcache=kv)
        sw = _scale_rows_f32(d["kvcache"]).flip(1).contiguous()  # row t/32 off by one
        kv2 = d["kvcache"].clone()
        kv2[:, 0, PAGE:] = sw.view(torch.float8_e4m3fn).reshape(kv2[:, 0, PAGE:].shape)
        out["k_scale_row_shift"] = cp(kvcache=kv2)
    else:
        out["k_scale_x2"] = cp(k_scale=d["k_scale"] * 2)
    kv = d["kvcache"].clone()
    for b, n in enumerate(d["kv_lens_total"].tolist()):
        ids = d["block_ids"][b, :(n + PAGE - 1) // PAGE].long()
        if len(ids) > 1:  # K (not V) read from the wrong pages
            kv[ids, 0] = d["kvcache"][ids.roll(1), 0]
    out["k_pages_shuffled"] = cp(kvcache=kv)
    if sq > 1:
        qs = d["q_scale"].reshape(-1, sq, d["q_scale"].shape[1]).clone()
        qs[:, [0, 1]] = qs[:, [1, 0]]
        out["q_scale_mtp_rows_swapped"] = cp(q_scale=qs.reshape(d["q_scale"].shape))
    out["causal_limit_plus_one"] = cp(kv_lens_total=d["kv_lens_total"] + 1)
    return out


DECODE_FAMILIES = [
    # (kind, temperature, k_per_token, lens, num_seq_q, hkv, hq); lens not page multiples, so
    # that the causal mutation has a slot to read
    ("peaked", 1.0, False, [300, 131, 77], 2, 2, 8),
    ("peaked", 4.0, False, [300, 131, 77], 2, 2, 8),
    ("peaked", 16.0, False, [300, 131, 77], 2, 2, 8),
    ("peaked", 4.0, True, [300, 131, 77], 2, 2, 8),
    ("peaked", 16.0, True, [300, 131, 77], 3, 1, 8),
    ("needle", 0.0, False, [200, 131, 70], 3, 2, 8),
    ("needle", 0.0, True, [200, 131, 70], 4, 2, 8),
    ("kscale", 0.0, True, [200, 131, 140], 2, 2, 8),
]


@pytest.mark.parametrize("fam", DECODE_FAMILIES, ids=lambda f: f"{f[0]}-T{f[1]}-kpt{int(f[2])}-sq{f[4]}")
def test_decode_exact_checks_discriminate(fam):
    kind, t, kpt, lens, sq, hkv, hq = fam
    d = make_decode_exact_inputs(kind, lens, sq, hkv, hq, k_per_token=kpt, temperature=t, seed=3)
    y, bound = decode_exact(d, sq, kpt)
    lossy = decode_lossy(d, sq, kpt)
    r = ox.grade(lossy, y, bound, lossy)
    assert r["ok_a"], f"lossy oracle outside B: {r}"
    assert r["rel_oracle"] < 0.1, r
    undetected = []
    for name, m in decode_mutations(d, sq, kpt).items():
        rm = ox.grade(decode_lossy(m, sq, kpt), y, bound, lossy)
        if rm["ok_a"] and rm["ok_b"]:
            undetected.append((name, rm))
    assert not undetected, undetected


# ------------------------------------------------------------------------------------------------
# prefill
# ------------------------------------------------------------------------------------------------
def prefill_lossy(d, kpt):
    return op.blocksparse_prefill(d["q"], d["kcache"], d["vcache"], d["qscale"], d["kscale"],
                                  d["vscale"], d["cu_seqlens_q"], d["seqlens_kv"], d["block_ids"],
                                  d["block_mask"], kpt)


def prefill_exact(d, kpt):
    return ox.prefill_fp8_exact(d["q"], d["kcache"], d["vcache"], d["qscale"], d["kscale"],
                                d["vscale"], d["cu_seqlens_q"], d["seqlens_kv"], d["block_ids"],
                                d["block_mask"], kpt)


def prefill_mutations(d, kpt):
    out = {}
    gen = torch.Generator().manual_seed(98)

    def cp(**kw):
        e = dict(d)
        e.update(kw)
        return e

    qf = d["q"].float()
    out["unrelated_q"] = cp(q=(torch.randn(qf.shape, generator=gen) * qf.std()).clamp(-440, 440)
                          .to(torch.float8_e4m3fn))  # finite codes: the scores must reject it
    out["zero_q"] = cp(q=torch.zeros_like(qf).to(torch.float8_e4m3fn))
    bm = d["block_mask"]
    out["reversed_q_heads"] = cp(q=d["q"].flip(1), qscale=d["qscale"].flip(1),
                                 block_mask=None if bm is None else bm.flip(1))
    out["k_scale_x2"] = cp(kscale=d["kscale"] * 2)
    if kpt:
        out["k_scale_row_shift"] = cp(kscale=d["kscale"].flip(1).contiguous())
    k = d["kcache"].clone()
    for b, n in enumerate(d["seqlens_kv"].tolist()):
        ids = d["block_ids"][b, :(n + PAGE - 1) // PAGE].long()
        if len(ids) > 1:
            k[ids] = d["kcache"][ids.roll(1)]
    out["k_pages_shuffled"] = cp(kcache=k)
    qs = d["qscale"].clone()
    qs[:, :, [0, 1]] = qs[:, :, [1, 0]]
    out["q_scale_rows_swapped"] = cp(qscale=qs)
    out["causal_limit_plus_one"] = cp(seqlens_kv=d["seqlens_kv"] + 1)
    if bm is not None:
        hidden = _skipped_tile(d)
        if hidden is not None:
            m2 = bm.clone()
            m2[hidden] = True
            out["skipped_tile_visited"] = cp(block_mask=m2)
    return out


def _skipped_tile(d):
    """First (b, q head, Q tile, KV tile) that the mask skips inside the causal extent."""
    bm = d["block_mask"]
    cu = d["cu_seqlens_q"].tolist()
    for b, nkv in enumerate(d["seqlens_kv"].tolist()):
        nq = cu[b + 1] - cu[b]
        for m in range((nq + 127) // 128):
            last = (nkv - nq + min(nq, (m + 1) * 128) - 1) // 128
            for h in range(bm.shape[1]):
                for n in range(min(last + 1, bm.shape[-1])):
                    if not bm[b, h, m, n]:
                        return (b, h, m, n)
    return None


PREFILL_FAMILIES = [
    # (kind, temperature or climb, k_per_token, q_lens, kv_lens, hq, hkv, skip)
    ("peaked", 1.0, False, [300, 150], [300, 330], 4, 2, 0.4),
    ("peaked", 4.0, False, [300, 150], [300, 330], 4, 2, 0.4),
    ("peaked", 16.0, True, [300, 150], [300, 330], 4, 2, 0.4),
    ("peaked", 4.0, True, [300, 150], [300, 330], 4, 2, None),
    ("sched", 0.70, False, [300, 150], [300, 330], 4, 1, 0.3),
    ("sched", 0.80, True, [300, 150], [300, 330], 4, 1, 0.3),
    ("sched", 20.0, False, [400, 130], [460, 400], 2, 1, 0.3),
    ("sched", -30.0, True, [400, 130], [460, 400], 2, 1, 0.3),
]


@pytest.mark.parametrize("fam", PREFILL_FAMILIES, ids=lambda f: f"{f[0]}-{f[1]}-kpt{int(f[2])}-skip{f[7]}")
def test_prefill_exact_checks_discriminate(fam):
    kind, t, kpt, ql, kl, hq, hkv, skip = fam
    kw = dict(temperature=t) if kind == "peaked" else dict(climb=t)
    d = make_prefill_exact_inputs(ql, kl, hq, hkv, skip, kpt, kind=kind, seed=5, **kw)
    y, bound = prefill_exact(d, kpt)
    lossy = prefill_lossy(d, kpt)
    r = ox.grade(lossy, y, bound, lossy)
    assert r["ok_a"], f"lossy oracle outside B: {r}"
    assert r["rel_oracle"] < 0.1, r
    undetected = []
    for name, m in prefill_mutations(d, kpt).items():
        rm = ox.grade(prefill_lossy(m, kpt), y, bound, lossy)
        if rm["ok_a"] and rm["ok_b"]:
            undetected.append((name, rm))
    assert not undetected, undetected


def test_prefill_dead_q_tile_is_nan_in_both():
    d = make_prefill_exact_inputs([300], [300], 2, 1, 0.0, False, seed=6, dead_tile=(0, 1, 1))
    y, bound = prefill_exact(d, False)
    lossy = prefill_lossy(d, False)
    assert torch.isnan(y[128:256, 1]).all() and not torch.isnan(y[:128]).any()
    assert ox.grade(lossy, y, bound, lossy)["ok_a"]


def test_exp2_poly_error_is_what_the_kernel_comment_states():
    # csrc/prefill_common.cuh documents a relative error of 7.5e-5 for exp2_poly_pair
    assert 5e-5 < ox.exp2_poly_rel_err() < 8e-5
