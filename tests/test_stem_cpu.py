"""Stem oracle (oracle/stem.py) on hand-worked cases, the operator surface, the wrappers' argument
checks, and simulated kernel bugs that each stage check must reject. CPU only."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import stem as os_
from synth import stem as ss

SCHEMAS = Path(__file__).resolve().parent / "golden" / "reference_schemas.json"
NAMES = ["stem_oam_prep_paged_kv", "stem_oam_prep_varlen_q", "stem_oam_gemm", "stem_tpd"]


def _bf16(vals):
    return torch.tensor(vals, dtype=torch.float32).to(torch.bfloat16)


def _mask_row(vals, budget_blocks, q_len=128, kv=None, alpha=1.0, initial=0, window=0):
    x = _bf16(vals)[None, None, None, :]
    kv = len(vals) * 128 if kv is None else kv
    args = [torch.tensor([v], dtype=torch.int32) for v in (q_len, kv, budget_blocks * 128)]
    return os_.tpd(x, *args, alpha=alpha, initial_blocks=initial, window_size=window)[0, 0, 0]


# ---- TPD hand cases --------------------------------------------------------------------------
def test_ordered_keys():
    k = os_.ordered_keys(_bf16([-1.0, -0.0, 0.0, 1.0, float("inf"), float("nan"), float("-inf")])
                         .view(torch.int16).numpy().astype(np.uint16))
    assert k[0] < k[1] < k[2] < k[3]  # -0 orders below +0
    assert list(k[4:]) == [0x7F] * 3


def test_tpd_ties_kept():
    # P = 3 blocks -> budget 3 (small regime); diag is the last column (window 0 still keeps it)
    m = _mask_row([5.0, 2.0, 2.0, 2.0, 1.0, 9.0], 3, kv=6 * 128, q_len=128)
    # top-3 threshold is 2.0 and every tie at 2.0 is kept; col 5 is the diagonal
    assert list(m) == [1, 1, 1, 1, 0, 1]


def test_tpd_signed_zero():
    m = _mask_row([-0.0, 0.0, -1.0, -2.0, -3.0, -4.0], 1, kv=6 * 128)
    assert list(m[:2]) == [0, 1]


def test_tpd_fewer_finite_than_budget():
    ninf = float("-inf")
    m = _mask_row([ninf, 1.0, float("nan"), 2.0, float("inf"), ninf, ninf, 0.5], 6, kv=8 * 128)
    # budget 6 covers the 3 finite values: all of them, never a non-finite one (+ the diagonal)
    assert list(m) == [0, 1, 0, 1, 0, 0, 0, 1]


def test_budget_regimes():
    assert os_.budget(0, 55) == 55
    assert os_.budget(10, 56) == int(np.float32(56) * np.float32(0.2)) + 30 == 41
    assert os_.budget(10, 160) == 46
    # decay: q_pos >= k; linear toward k * alpha over the prompt
    assert os_.budget(200, 300, alpha=0.5) < os_.budget(60, 300, alpha=0.5) <= 60
    assert os_.budget(299, 300, alpha=0.5) == 30
    assert os_.budget(299, 300, alpha=1.0) == 60


def test_budget_fma_matters_somewhere():
    diff = [(P, q) for P in range(56, 400) for q in range(P)
            if os_.budget(q, P, 0.3) != os_.budget(q, P, 0.3, fma=False)]
    assert diff, "the single-rounding decay never matters: the fma test would be vacuous"


def test_round_f32_is_single_rounding():
    from fractions import Fraction
    assert os_._round_f32(Fraction(1, 3)) == np.float32(1 / 3)
    half = Fraction(1) + Fraction(1, 2 ** 24)  # tie between 1 and 1 + 2^-23 -> even (1)
    assert os_._round_f32(half) == np.float32(1.0)


# ---- surface and argument checks ---------------------------------------------------------------
def test_schemas_and_exports(hpc):
    from test_api_surface import _canon

    ref = json.loads(SCHEMAS.read_text())
    for n in NAMES:
        assert _canon(getattr(torch.ops.hpc, n).default._schema) == _canon("hpc::" + ref[n])
    for f in NAMES + ["stem_paged_kv"]:
        assert callable(getattr(hpc, f))


def test_launcher_rejects_bad_arguments(hpc):
    lib = hpc._ffi.lib
    args = [None] * 8 + [1, 128, 128, 2, 4, 16, 4, 128, 16, 0.3, 1, 8, 0, 0, 0, 0, 0, 0, None, None]
    assert lib.hpc_stem_oam_prep_paged_kv_qpertoken_perhead_kvpertensor_dim128_async(*args) != 0
    assert b"32 or 64" in lib.hpc_last_error()
    a = list(args)
    a[9] = 64
    a[13] = 64
    assert lib.hpc_stem_oam_prep_paged_kv_qpertoken_perhead_kvpertensor_dim128_async(*a) != 0
    assert b"dim_qk=64" in lib.hpc_last_error()
    a = list(args)
    a[13], a[15] = 64, 64
    assert lib.hpc_stem_oam_prep_paged_kv_qpertoken_perhead_kvpertensor_dim128_async(*a) != 0
    assert b"stem_block_size=128" in lib.hpc_last_error()
    tpd = [None] * 5 + [1, 1, 1, 40000, 128, 1.0, 4, 4, 0.2, 30, 0.1, 30, None]
    assert lib.hpc_stem_tpd_async(*tpd) != 0 and b"32768" in lib.hpc_last_error()
    gemm = [None] * 6 + [1, 6, 4, 1, 1, 128, 16, 1, None]
    assert lib.hpc_stem_oam_gemm_dim128_async(*gemm) != 0 and b"multiple" in lib.hpc_last_error()


def test_wrappers_reject_bad_input(hpc):
    # the op implementations check their arguments before the device, so CPU tensors reach each check
    from hpc import stem as hs

    i32 = torch.zeros(1, dtype=torch.int32)

    def raises(fn, *a, match):
        with pytest.raises(RuntimeError, match=match):
            fn(*a)

    raises(hs._tpd_impl, torch.zeros(1, 1, 1, 40000, dtype=torch.bfloat16), i32, i32, i32, 128, 1.0,
           4, 4, 0.2, 30, 0.1, 30, match="exceeds 32768")
    raises(hs._tpd_impl, torch.zeros(1, 1, 1, 8, dtype=torch.bfloat16), i32, i32, i32, 64, 1.0,
           4, 4, 0.2, 30, 0.1, 30, match="block_size must be 128")
    q = torch.zeros(1, 2, 4, 2048, dtype=torch.bfloat16)
    k = torch.zeros(1, 2, 4, 1024, dtype=torch.bfloat16)
    raises(hs._gemm_impl, q, k, torch.zeros(1, 2, 4), i32, i32, 128, 16, True, match="kFlatDim mismatch")
    raises(hs._gemm_impl, q, q, torch.zeros(1, 2, 4), i32, i32, 64, 16, True,
           match="stem_block_size=128")
    raises(hs._gemm_impl, q, q[:, :, :3].contiguous(), torch.zeros(1, 2, 4), i32, i32, 128, 16, True,
           match="vbias shape")
    raises(hs._gemm_impl, torch.zeros(1, 3, 4, 2048, dtype=torch.bfloat16), q, torch.zeros(1, 2, 4),
           i32, i32, 128, 16, True, match="divisible")
    ids = torch.zeros(1, 4, dtype=torch.int32)
    for page in (16, 128):
        kc = torch.zeros(4, page, 2, 128, dtype=torch.float8_e4m3fn)
        raises(hs._prep_paged_kv_impl, kc, kc, torch.ones(1), torch.ones(1), ids, i32, 0.3, 128, 16, 1,
               match="must be 32 or 64")
    kc = torch.zeros(4, 64, 2, 64, dtype=torch.float8_e4m3fn)
    raises(hs._prep_paged_kv_impl, kc, kc, torch.ones(1), torch.ones(1), ids, i32, 0.3, 128, 16, 1,
           match="dim_qk=64")
    kc = torch.zeros(4, 64, 2, 128, dtype=torch.float8_e4m3fn)
    raises(hs._prep_paged_kv_impl, kc, kc, torch.ones(1), torch.ones(1), ids, i32, 0.3, 256, 16, 1,
           match="stem_block_size=128")
    raises(hs._prep_paged_kv_impl, kc, kc, torch.ones(1), torch.ones(1), ids,
           torch.tensor([300], dtype=torch.int32), 0.3, 128, 16, 1, match="exceed the block table")
    raises(hs._prep_paged_kv_impl, kc, kc, torch.ones(1), torch.ones(1), ids, i32, 0.3, 128, 16, 0,
           match="quant_type 0 takes kscale")
    qf = torch.zeros(10, 2, 128, dtype=torch.float8_e4m3fn)
    cu = torch.tensor([0, 10], dtype=torch.int32)
    raises(hs._prep_varlen_q_impl, qf, torch.ones(1, 2, 8), torch.tensor([10], dtype=torch.int32), cu,
           128, 16, match="exceed qscale")
    raises(hs._prep_varlen_q_impl, torch.zeros(10, 2, 64, dtype=torch.float8_e4m3fn), torch.ones(1, 2, 16),
           torch.tensor([10], dtype=torch.int32), cu, 128, 16, match="dim_qk=128")
    # CPU tensors that pass every argument check are refused as not being on the GPU
    raises(hs._tpd_impl, torch.zeros(1, 1, 1, 8, dtype=torch.bfloat16), i32, i32, i32, 128, 1.0,
           4, 4, 0.2, 30, 0.1, 30, match="CUDA tensors")


# ---- the KV-prep oracle against the reference's own functions (tests/golden/make_golden_stem.py) ----
@pytest.mark.parametrize("tag", ["q0_p32", "q1_p64", "q0_p64"])
def test_kv_prep_oracle_matches_reference_golden(tag):
    z = np.load(Path(__file__).resolve().parent / "golden" / f"stem_kvprep_{tag}.npz")
    page, quant = (int(v) for v in z["meta"])
    kc = torch.from_numpy(z["kcache"]).view(torch.float8_e4m3fn)
    vc = torch.from_numpy(z["vcache"]).view(torch.float8_e4m3fn)
    lens = torch.from_numpy(z["kv_seq_lens"])
    kv = os_.kv_prep(kc, vc, torch.from_numpy(z["kscale"]), torch.from_numpy(z["vscale"]),
                     torch.from_numpy(z["kv_indices"]), lens, 0.3, quant)
    gk = torch.from_numpy(z["kflat"]).view(torch.bfloat16).double().numpy()
    for b, o in enumerate(kv):
        nkb = o["vbias"].shape[1]
        # the reference scales each row before summing in fp32: it may land on the neighbouring bf16
        # (per-row products rounded, then an fp32 sum), so allow that order's error
        acc = 2 * os_.SAMPLES * os_.U * o["kflat_abs"] + os_.U * np.abs(o["kflat"])
        tol = 2 * os_.half_ulp_bf16(np.abs(o["kflat"]) + acc) + acc
        assert not _fails(gk[b, :, :nkb], o["kflat"], tol), f"kflat b{b}"
        assert not _fails(z["vbias"][b, :, :nkb], o["vbias"], 2 * o["vbias_bound"] + 1e-6), f"vbias b{b}"


# ---- simulated bugs: each fails its stage check on the synth inputs ------------------------------
@pytest.fixture(scope="module")
def case():
    d = ss.make_inputs([300, 77], [1000, 3100], 4, 2, 64, "nhd", 0, seed=5)
    kv = os_.kv_prep(d["kcache"], d["vcache"], d["kscale"], d["vscale"], d["kv_indices"],
                     d["kv_seq_lens"], 0.3, 0)
    return d, kv


def _fails(x, ref, bound):
    return bool((~(np.abs(x - ref) <= bound)).any())


def _bf16r(x):
    return torch.from_numpy(np.ascontiguousarray(x)).float().to(torch.bfloat16).double().numpy()


def test_bug_group_order_not_reversed(case):
    d, kv = case
    k = kv[1]["kflat"].reshape(2, -1, 16, 128)[:, :, ::-1].reshape(2, -1, 2048)
    assert _fails(_bf16r(k), kv[1]["kflat"], kv[1]["kflat_bound"])


def test_bug_kscale_dropped(case):
    d, kv = case
    ones = torch.ones_like(d["kscale"])
    kv0 = os_.kv_prep(d["kcache"], d["vcache"], ones, d["vscale"], d["kv_indices"],
                      d["kv_seq_lens"], 0.3, 0)
    assert _fails(_bf16r(kv0[1]["kflat"]), kv[1]["kflat"], kv[1]["kflat_bound"])


def test_bug_poisoned_tail_summed(case):
    # a kernel that reads one row past kv_len sums the NaN poison of the page tail into kflat
    d, kv = case
    longer = d["kv_seq_lens"] + 1
    bad = os_.kv_prep(d["kcache"], d["vcache"], d["kscale"], d["vscale"], d["kv_indices"], longer, 0.3, 0)
    assert _fails(_bf16r(bad[1]["kflat"]), kv[1]["kflat"], kv[1]["kflat_bound"])


def _vbias_variant(d, **kw):
    from oracle.stem import _pages

    b, h = 1, 0
    n = int(d["kv_seq_lens"][b])
    v = _pages(d["vcache"], d["kv_indices"][b], n, h)
    return os_.vbias_stats(v, float(d["vscale"][h]), os_.cdiv(n, 128), 0.3, **kw)


def test_bug_biased_std(case):
    d, kv = case
    ref, bnd = _vbias_variant(d)
    bad, _ = _vbias_variant(d, ddof=0)
    assert _fails(bad, ref, bnd)


def test_bug_padding_excluded_from_vbias(case):
    d, kv = case
    ref, bnd = _vbias_variant(d)
    bad, _ = _vbias_variant(d, pad_rows=False)
    assert _fails(bad, ref, bnd)


def test_bug_floor_causal_offset():
    # chunked: kv - q = 3100 - 300 is not a multiple of 128, so floor and ceil differ by one block
    g = torch.Generator().manual_seed(3)
    ql, kl = torch.tensor([300], dtype=torch.int32), torch.tensor([3100], dtype=torch.int32)
    qf = torch.randn(1, 2, 3, 2048, generator=g).to(torch.bfloat16)
    kf = torch.randn(1, 1, 25, 2048, generator=g).to(torch.bfloat16)
    y, bound, dead = os_.gemm(qf, kf, torch.zeros(1, 1, 25), ql, kl)
    floor_dead = os_.neg_inf_mask(300, 3100, 3, 25, offset=(3100 - 300) // 128)
    kernel = np.where(floor_dead[None, None], -np.inf, y)  # the simulated kernel's logits
    assert not np.array_equal(np.isneginf(kernel), dead)  # the GPU test's -inf check


def _synth_logits(seed=9):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(1, 2, 10, 80, generator=g).to(torch.bfloat16)
    ql = torch.tensor([10 * 128 - 3], dtype=torch.int32)
    kl = torch.tensor([80 * 128 - 50], dtype=torch.int32)
    return x, ql, kl, kl.clone()


def test_bug_budget_off_by_one():
    x, ql, kl, p = _synth_logits()
    good = os_.tpd(x, ql, kl, p, alpha=0.5)
    bad = os_.tpd(x, ql, kl, p, alpha=0.5, budget_fn=lambda *a: os_.budget(*a) + 1)
    assert not np.array_equal(good, bad)


def test_bug_non_fma_decay():
    P, q = next((P, q) for P in range(56, 400) for q in range(P)
                if os_.budget(q, P, 0.3) != os_.budget(q, P, 0.3, fma=False))
    x = torch.randn(1, 1, q + 1, P, generator=torch.Generator().manual_seed(1)).to(torch.bfloat16)
    args = [torch.tensor([v], dtype=torch.int32) for v in (128 * (q + 1), 128 * P, 128 * P)]
    good = os_.tpd(x, *args, alpha=0.3)
    bad = os_.tpd(x, *args, alpha=0.3,
                  budget_fn=lambda qp, PP, *a: os_.budget(qp, PP, *a, fma=False))
    assert not np.array_equal(good, bad)


def test_bug_float_compare_instead_of_ordered_keys():
    # comparing the raw bf16 bits as unsigned integers puts every negative value above the positives
    x, ql, kl, p = _synth_logits()
    good = os_.tpd(x, ql, kl, p, alpha=0.5)
    raw = x.view(torch.int16).numpy().astype(np.uint16)
    orig = os_.ordered_keys
    try:
        os_.ordered_keys = lambda bits: np.asarray(bits, dtype=np.int64) | 0x80
        bad = os_.tpd(torch.from_numpy(raw.view(np.int16)).view(torch.bfloat16), ql, kl, p, alpha=0.5)
    finally:
        os_.ordered_keys = orig
    assert not np.array_equal(good, bad)


def _tpd_keep_exactly_budget(x, ql, kl, prompt, alpha):
    """A TPD that keeps exactly `budget` columns per row (ties at the threshold broken by column
    index) instead of every column tied with the threshold: the simulated bug."""
    bits = x.contiguous().view(torch.int16).numpy().astype(np.uint16)
    B, H, max_qb, max_kb = bits.shape
    mask = np.zeros(bits.shape, dtype=np.uint8)
    for b in range(B):
        qi, ki = os_.cdiv(int(ql[b]), 128), os_.cdiv(int(kl[b]), 128)
        off = os_.causal_offset(int(ql[b]), int(kl[b]))
        P = os_.cdiv(int(prompt[b]), 128)
        cols = np.arange(ki)
        for qr in range(qi):
            bud = os_.budget(qr + off, P, alpha)
            diag = min(qr + off, ki - 1)
            fixed = (cols < 4) | ((cols <= diag) & (cols > diag - 4)) | (cols == diag)
            for h in range(H):
                keys = os_.ordered_keys(bits[b, h, qr, :ki])
                order = np.lexsort((cols, -keys))  # value desc, then column asc
                top = np.zeros(ki, dtype=bool)
                fin = order[keys[order] != os_.NON_FINITE][:max(bud, 0)]
                top[fin] = True
                mask[b, h, qr, :ki] = (top | fixed).astype(np.uint8)
    return mask


def test_bug_ties_broken_by_count():
    x = ss.adversarial_logits(1, 2, 9, 300, seed=4)  # many ties at every level
    ql = torch.tensor([9 * 128], dtype=torch.int32)
    kl = torch.tensor([300 * 128], dtype=torch.int32)
    good = os_.tpd(x, ql, kl, kl, alpha=0.5)
    bad = _tpd_keep_exactly_budget(x, ql, kl, kl, 0.5)
    assert not np.array_equal(bad, good)  # the GPU test's bit-exact TPD check
