"""The exact check of RoPE + QK-norm + paged KV store can tell (CPU only).

CASES is the case list tests/test_rope_exact_gpu.py runs through both hpc.rope_norm_store_kv and
hpc.rope_norm_store_kv_fp8, each on the cache path and with the out_q / out_k / out_v bypass.
For every case and call the fp32 emulation of the kernel that call launches
(oracle.rope_exact.launch_path, a restatement of csrc/rope.cu launch()) passes
oracle.rope_exact.grade with no unexplained difference, and every simulated bug of
oracle.rope_exact.MUTATIONS the case can express fails it. The case list is checked to reach
every kernel instantiation in bf16 and FP8, both V paths of the generic kernel and a d128 unit
that holds only some of its heads; the fp64 oracle is pinned to the reference function's goldens.
"""
import numpy as np
import pytest

from oracle import rope_exact as ore
from synth import rope as sr
from test_oracle_rope import load_rope

_QUANT = [(1, 448.0), (1, 224.0), (2, 100.5), (1, 100.5), (2, 224.0), (2, 448.0)]


def _case(name, hq, hkv, dqk, dv, page, layout, mode, policy, **kw):
    c = dict(name=name, hq=hq, hkv=hkv, dqk=dqk, dv=dv, page=page, layout=layout, mode=mode,
             policy=policy, seed=len(name) * 97 + page + dqk, misaligned=())
    c.update(kw)
    return c


CASES = [
    _case("d128-8x1-decode", 8, 1, 128, 128, 64, "split", "decode", 0, mtp=0, batch=5),
    _case("d128-28x4-prefill", 28, 4, 128, 128, 16, "combined", "prefill", 1),
    _case("d128-32x8-decode", 32, 8, 128, 128, 32, "combined", "decode", 2, mtp=1, batch=6),
    _case("d128-64x8-long", 64, 8, 128, 128, 24, "split", "decode", 1, mtp=3, batch=3, long=True),
    _case("d128-32x8-rotary", 32, 8, 128, 128, 64, "split", "prefill", 2, table="rotary"),
    _case("k1-d64-8x1", 8, 1, 64, 64, 16, "split", "prefill", 2),
    _case("k1-d96-28x4", 28, 4, 96, 96, 24, "combined", "decode", 1, mtp=2, batch=4),
    _case("k2-d192-32x8", 32, 8, 192, 192, 32, "split", "prefill", 0),
    _case("k2-d256-8x1", 8, 1, 256, 256, 64, "combined", "decode", 2, mtp=1, batch=5),
    _case("k4-d320-28x4", 28, 4, 320, 320, 16, "split", "decode", 1, mtp=0, batch=9),
    _case("d128-dv64", 32, 8, 128, 64, 32, "split", "prefill", 1),
    _case("d128-dv256", 8, 1, 128, 256, 16, "split", "decode", 2, mtp=2, batch=3),
    _case("k1-scalar-v", 8, 2, 64, 70, 24, "split", "prefill", 1),
    _case("fallback-qkv+4", 32, 8, 128, 128, 64, "split", "decode", 1, mtp=1, batch=4,
          misaligned=("qkv",)),
    _case("fallback-qnorm+4", 8, 1, 128, 128, 16, "split", "prefill", 2, misaligned=("q_norm_w",)),
    _case("fallback-outk+4", 28, 4, 128, 128, 32, "combined", "decode", 1, mtp=3, batch=2,
          misaligned=("out_k",)),
]
for _i, _c in enumerate(CASES):
    _c["quant_policy"], _c["upper_max"] = _QUANT[_i % len(_QUANT)]


def case_id(c):
    return c["name"]


def fp8_args(c):
    return dict(k_scale=0.37, v_scale=0.21, quant_policy=c["quant_policy"], upper_max=c["upper_max"],
                q_scale_inv=9.3)


def misaligned(c, bypass):
    """The pointers of the call that are not 16-byte aligned (out_k only exists on the bypass)."""
    return tuple(m for m in c["misaligned"] if bypass or m != "out_k")


def path_of(c, inp, fp8, bypass):
    return ore.launch_path(inp["geom"], fp8, misaligned(c, bypass))


def sentinel_flat(inp, fp8):
    n = inp["geom"]["flat"]
    return np.full(n, sr.FP8_SENTINEL, np.uint8) if fp8 else np.full(n, sr.BF16_SENTINEL, np.uint16)


_INPUTS = {}


def inputs(c):
    if c["name"] not in _INPUTS:
        _INPUTS[c["name"]] = sr.make_exact_inputs(c)
    return _INPUTS[c["name"]]


def _emulated(c, fp8, bypass=False, mutation=None):
    inp = inputs(c)
    before = sentinel_flat(inp, fp8)
    fa = fp8_args(c) if fp8 else None
    out = ore.emulate(inp, fp8, path_of(c, inp, fp8, bypass), mutation, fa, bypass, before)
    return ore.grade(inp, out, fp8, path_of(c, inp, fp8, bypass), fa, before)


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_rope_exact_checks_discriminate(c, fp8):
    for bypass in (False, True):
        res = _emulated(c, fp8, bypass)
        assert not ore.failed(res), (bypass, res)
    inp = inputs(c)
    undetected = []
    for m in ore.mutations_for(inp, fp8, fp8_args(c)):
        res = _emulated(c, fp8, mutation=m)
        if not ore.failed(res):
            undetected.append(m)
    assert not undetected, undetected


def _v_paths(c, inp, fp8, bypass):
    rows = inp["qkv"].shape[0]
    off = 4 if "qkv" in misaligned(c, bypass) else 0
    vec = ore.generic_v_vector_rows(inp["geom"], fp8, rows, off, out_v=bypass)
    pos, _ = ore.positions(inp["num_seqlen"], inp["q_index"], rows)
    return {bool(v) for v in vec[pos >= 0]}


def test_rope_exact_cases_cover_the_launch_paths():
    """Every instantiation of launch() in bf16 and FP8, both V paths of the generic kernel, a
    d128 unit with only some of its 8 heads, the combined cache, every page size, GQA ratio,
    head dim and request shape the cases claim."""
    for fp8 in (False, True):
        paths, vpaths, partial = set(), set(), False
        for c in CASES:
            inp = inputs(c)
            for bypass in (False, True):
                kind, kch = path_of(c, inp, fp8, bypass)
                paths.add((kind, kch))
                if kind == "generic":
                    vpaths |= _v_paths(c, inp, fp8, bypass)
                else:
                    partial |= c["hq"] % 8 != 0 or c["hkv"] % 8 != 0
        assert paths == {("d128", 1), ("generic", 1), ("generic", 2), ("generic", 4)}, (fp8, paths)
        assert vpaths == {True, False}, fp8
        assert partial
    for m in ("qkv", "q_norm_w", "out_k"):
        c = next(c for c in CASES if m in c["misaligned"])
        assert c["dqk"] == 128 and path_of(c, inputs(c), False, True) == ("generic", 1)
    assert {c["page"] for c in CASES} == {16, 24, 32, 64}
    assert {(c["hq"], c["hkv"]) for c in CASES} >= {(8, 1), (28, 4), (32, 8), (64, 8)}
    assert {c["dqk"] for c in CASES} >= {64, 96, 128, 192, 256, 320}
    assert {c["dv"] for c in CASES if c["dqk"] == 128} >= {64, 128, 256}
    assert {c["mtp"] for c in CASES if c["mode"] == "decode"} == {0, 1, 2, 3}
    assert {c["layout"] for c in CASES} == {"split", "combined"}
    assert {(qp, um) for c in CASES for qp, um in [(c["quant_policy"], c["upper_max"])]} == set(_QUANT)
    assert any(c.get("table") == "rotary" for c in CASES)
    for c in CASES:
        inp = inputs(c)
        q_len = np.diff(inp["q_index"].numpy())
        if c["mode"] == "prefill":  # zero-row requests between others, one with no tokens at all
            assert (q_len[1:-1] == 0).any() and (inp["num_seqlen"].numpy() == 0).any()
        else:  # padded to 8 requests and rows
            assert inp["qkv"].shape[0] % 8 == 0 and inp["num_seqlen"].shape[0] % 8 == 0
        pos, _ = ore.positions(inp["num_seqlen"], inp["q_index"], inp["qkv"].shape[0])
        if c.get("long"):
            assert pos.max() > 65536
    for m in ore.MUTATIONS:  # every mutation is checked on some case
        assert any(m in ore.mutations_for(inputs(c), True, fp8_args(c)) for c in CASES), m


@pytest.mark.parametrize("name", ["rope_prefill_p2.npz", "rope_decode_p1.npz"])
def test_rope_exact_oracle_matches_reference_goldens(name):
    """The reference function (torch fp32) lies within the fp64 oracle's bound for a sum of D
    squares in any order and a rsqrt of two roundings, up to explained bf16 flips, on Q and on
    the cache it writes."""
    d, out, (num_req, is_prefill, mtp, hq, hkv, policy) = load_rope(name)
    kc, vc = d["kcache"], d["vcache"]
    D, dv, page = kc.shape[3], vc.shape[3], kc.shape[1]
    n = kc.shape[0]
    geom = dict(hq=hq, hkv=hkv, dqk=D, dv=dv, page=page, layout="split", num_pages=n,
                k_off=0, v_off=n * page * hkv * D, k_stride=page * hkv * D, v_stride=page * hkv * dv)
    inp = dict(qkv=d["qkv"], cos_sin=d["cos_sin"], num_seqlen=d["num_seqlen"], q_index=d["q_index"],
               kv_indices=d["kv_indices"], q_norm_w=d["q_norm_w"], k_norm_w=d["k_norm_w"], geom=geom,
               is_prefill=is_prefill, policy=policy)
    rows = int(d["q_index"][-1])
    inp["qkv"] = d["qkv"][:rows]
    before = np.concatenate([ore.bits(kc).ravel(), ore.bits(vc).ravel()])
    after = np.concatenate([ore.bits(out["kcache"]).ravel(), ore.bits(out["vcache"]).ravel()])
    # torch's mean of D squares: at most D - 1 + 1 roundings per square -> sum_terms of kch = D/4
    res = ore.grade(inp, dict(q=ore.bits(out["q"]), cache=after), False, ("generic", D // 4), None,
                    before)
    assert not ore.failed(res), res
    assert res["flips_q"] + res["flips_k"] < 0.01 * (rows * (hq + hkv) * D), res
