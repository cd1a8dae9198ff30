"""bf16 prefill without a GPU: the oracle against the reference's own outputs, the exact check
against brute force and against the kernel bugs it must catch, the op schemas, and the launchers'
argument checks."""
import json
import math
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import prefill_bf16 as ob
from synth import prefill_bf16 as sb

GOLDEN = Path(__file__).resolve().parent / "golden"


def _bf16(a):
    return torch.from_numpy(a).view(torch.bfloat16)


# ------------------------------------------------------------------------------------------------
# oracle vs the reference's functions
# ------------------------------------------------------------------------------------------------
def test_golden_dense():
    z = np.load(GOLDEN / "prefill_bf16_dense.npz")
    out = ob.varlen_prefill(_bf16(z["q"]), _bf16(z["k"]), _bf16(z["v"]),
                            torch.from_numpy(z["cu_seqlens_q"]))
    torch.testing.assert_close(out, torch.from_numpy(z["out"]), atol=2e-6, rtol=1e-5)


@pytest.mark.parametrize("tag", ["kv_nhd_bs16", "kv_hnd_bs64"])
def test_golden_kvcache(tag):
    z = np.load(GOLDEN / f"prefill_bf16_{tag}.npz")
    hq, hkv, page, hnd = (int(x) for x in z["meta"])
    kc, vc = _bf16(z["kcache"]), _bf16(z["vcache"])
    if hnd:  # the same logical cache seen through head-major storage
        kc, vc = (t.transpose(1, 2).contiguous().transpose(1, 2) for t in (kc, vc))
    assert kc.shape[1] == page and kc.shape[2] == hkv
    out = ob.kvcache_prefill(_bf16(z["q"]), kc, vc, torch.from_numpy(z["cu_seqlens_q"]),
                             torch.from_numpy(z["block_ids"]), torch.from_numpy(z["seqlens_kv"]))
    torch.testing.assert_close(out, torch.from_numpy(z["out"]), atol=2e-6, rtol=1e-5)
    # the exact reference computes the same function
    y, _ = ob.paged_exact(_bf16(z["q"]), kc, vc, torch.from_numpy(z["cu_seqlens_q"]),
                          torch.from_numpy(z["block_ids"]), torch.from_numpy(z["seqlens_kv"]))
    torch.testing.assert_close(y.float(), torch.from_numpy(z["out"]), atol=2e-5, rtol=1e-4)


# ------------------------------------------------------------------------------------------------
# exact reference vs brute force
# ------------------------------------------------------------------------------------------------
def _brute(q, keys, vals, nkv):
    """fp64, one request: q [sq, Hq, D], keys / vals [nkv, Hkv, D], bottom-right causal."""
    sq, hq, d = q.shape
    g = hq // keys.shape[1]
    out = torch.empty(sq, hq, d, dtype=torch.float64)
    for h in range(hq):
        for i in range(sq):
            n = nkv - sq + i + 1
            s = keys[:n, h // g].double() @ q[i, h].double() / math.sqrt(d)
            w = torch.exp(s - s.max())
            out[i, h] = (w[:, None] * vals[:n, h // g].double()).sum(0) / w.sum()
    return out


@pytest.mark.parametrize("case", [sb.GRID[0], sb.GRID[3]], ids=sb.case_id)
def test_exact_matches_brute_force(case):
    d = sb.make_exact_case(case, "peaked")
    cu = d["cu_seqlens_q"]
    if d["op"] == "dense":
        y, bound = ob.dense_exact(d["q"], d["k"], d["v"], cu)
    else:
        y, bound = ob.paged_exact(d["q"], d["kcache"], d["vcache"], cu, d["block_ids"],
                                  d["seqlens_kv"])
    assert bool(torch.isfinite(bound).all()) and bool((bound > 0).all())
    for b in range(cu.numel() - 1):
        s0, s1 = int(cu[b]), int(cu[b + 1])
        if s1 == s0:
            continue
        if d["op"] == "dense":
            keys, vals, nkv = d["k"][s0:s1], d["v"][s0:s1], s1 - s0
        else:
            nkv = int(d["seqlens_kv"][b])
            ids = d["block_ids"][b, :(nkv + case["page"] - 1) // case["page"]]
            keys = ob.gather_pages(d["kcache"], ids, nkv)
            vals = ob.gather_pages(d["vcache"], ids, nkv)
        ref = _brute(d["q"][s0:s1], keys, vals, nkv)
        assert float((y[s0:s1] - ref).abs().max()) < 1e-9


# ------------------------------------------------------------------------------------------------
# the check passes the lossy oracle and rejects each kernel bug, on the GPU grid's own cases
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", sb.GRID, ids=sb.case_id)
def test_check_rejects_mutations(case):
    inputs = {kind: sb.make_exact_case(case, kind) for kind in sb.KINDS}
    for kind, d in inputs.items():
        r = ob.check(ob.mutant(d, None), d)
        assert r["ok_a"] and r["ok_b"], f"{kind}: the lossy oracle fails its own check: {r}"
    for m in ob.MUTATIONS:
        if not sb.applicable(case, m):
            continue
        caught = []
        for kind, d in inputs.items():
            r = ob.check(ob.mutant(d, m), d)
            caught.append(not (r["ok_a"] and r["ok_b"]))
        assert all(caught), f"mutation {m} passes the check for {dict(zip(sb.KINDS, caught))}"


def test_every_mutation_is_exercised():
    for m in ob.MUTATIONS:
        assert any(sb.applicable(c, m) for c in sb.GRID), m


# ------------------------------------------------------------------------------------------------
# schemas
# ------------------------------------------------------------------------------------------------
def test_schemas_match_reference(hpc):
    from test_api_surface import SCHEMAS, _canon

    ref = json.loads(SCHEMAS.read_text())
    for name in ("attention_prefill_bf16", "attention_with_kvcache_prefill_bf16"):
        mine = _canon(getattr(torch.ops.hpc, name).default._schema)
        assert mine == _canon("hpc::" + ref[name]), name
        assert callable(getattr(hpc, name))


# ------------------------------------------------------------------------------------------------
# launcher argument checks (no CUDA call is made before them)
# ------------------------------------------------------------------------------------------------
P = 4096  # an aligned address that is never dereferenced


def _dense(lib, dim=128, hq=8, hkv=2, ldq=1024):
    return lib.hpc_attention_prefill_bf16_async(P, P, P, P, P, P, 2, 100, 64, dim, dim, hq, hkv,
                                                hq * 128, ldq, hkv * 128, hkv * 128, None)


def _paged(lib, dim=128, hq=8, hkv=2, bs=64, tok=256):
    return lib.hpc_attention_with_kvcache_prefill_bf16_async(
        P, P, P, P, P, P, P, 2, 100, 64, dim, dim, hq, hkv, 10, bs, 4, hq * 128, hq * 128,
        bs * hkv * 128, tok, 128, bs * hkv * 128, tok, 128, None)


@pytest.mark.parametrize("call, text", [
    (lambda lib: _paged(lib, bs=48), "blocksize must be 16, 32 or 64"),
    (lambda lib: _paged(lib, dim=64), "head dim must be 128"),
    (lambda lib: _dense(lib, dim=64), "head dim must be 128"),
    (lambda lib: _paged(lib, hq=6, hkv=4), "multiple of num_head_kv"),
    (lambda lib: _dense(lib, hq=6, hkv=4), "multiple of num_head_kv"),
    (lambda lib: _paged(lib, tok=100), "multiples of 16 bytes"),
    (lambda lib: _dense(lib, ldq=1020), "multiples of 16 bytes"),
])
def test_launcher_rejects(hpc, call, text):
    lib = hpc._ffi.lib
    assert call(lib) == 1  # HPC_ERR_UNSUPPORTED
    msg = lib.hpc_last_error().decode()
    assert text in msg and "prefill_bf16" in msg, msg

