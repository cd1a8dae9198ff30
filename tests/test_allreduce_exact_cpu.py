"""The fused AllReduce + residual + RMSNorm checker (oracle.allreduce_exact) on the CPU: it agrees
with the reference's own arithmetic where both round once, it accepts an fp32 emulation of the
kernels in their summation order on every family and block shape, it rejects simulated bugs the
old atol = rtol = 0.1 comparison let through, and its Lamport workspace model is consistent."""
import numpy as np
import pytest
import torch

from oracle import allreduce as oa
from oracle import allreduce_exact as ox
from synth import allreduce as sa


def _case_args(c):
    return c["xs"], c["residual"], c["weight"], c["eps"]


def test_dispatch_tables_cover_every_instantiation():
    for kernel, table in (("ht", ox.HT_TABLE), ("ll", ox.LL_TABLE)):
        got = {ox.shape_of(h, kernel) for h in sa.HIDDENS}
        assert got == {(nvec, th) for _, nvec, th in table}, kernel


@pytest.mark.parametrize("W", [1, 2, 3, 4, 8])
def test_reference_against_pinned_oracle(W):
    """W <= 2: the pinned oracle rounds the sum once too, so out_residual is identical and out
    differs only where the checker allows either neighbour. W >= 3: its bf16 running sum rounds
    W - 1 times; every element where it differs from the exact reference is one the checker flags."""
    xs, res, w, n_pad = oa.make_inputs(W, 77, 7168)
    rr, ry = oa.allreduce_rmsnorm(xs, res, w, 1e-6)
    er, ey = ox.reference(xs, res, w, 1e-6)
    c = ox.check(rr, ry, xs, res, w, 1e-6)
    diff = (ox.f64(rr) != er) | (ox.f64(ry) != ey)
    flagged = c["bad_mask"] | c["amb_mask"]
    assert not (diff & ~flagged).any()
    if W <= 2:
        assert np.array_equal(ox.f64(rr), er)
        assert c["ok"], ox.summary(f"oracle W{W}", c)
    else:
        assert not c["ok"] and c["bad_res"] > 0


@pytest.mark.parametrize("H", sa.HIDDENS)
@pytest.mark.parametrize("kernel", ["ht", "ll"])
def test_emulation_passes_every_family(kernel, H):
    """The fp32 emulation in the kernel's order passes: the accepted set is not too tight."""
    T = 3 if H >= 16384 else 7
    for fam in sa.FAMILIES:
        for W in (1, 2, 3, 8):
            for eps in (sa.EPS if fam == "eps" else sa.EPS[:1]):
                c = sa.make_case(fam, W, T, H, seed=1, eps=eps)
                r, y = ox.emulate(*_case_args(c), kernel=kernel)
                res = ox.check(r, y, *_case_args(c), kernel=kernel)
                assert res["ok"], ox.summary(f"{kernel} {fam} W{W} T{T} H{H}", res)
                if fam in ("exact", "signature"):
                    assert res["amb_res"] == 0


# cases on which each simulated bug must fail the exact check
MUTANT_CASES = [("exact", 4, 7, 7168), ("cancel", 4, 7, 1024), ("eps", 2, 10, 7168),
                ("signature", 8, 7, 264), ("random", 4, 7, 7168)]


def test_mutants_fail_the_exact_check_and_pass_the_old_one():
    rows = []
    xs, res, w, _ = oa.make_inputs(4, 77, 7168)
    rr, ry = oa.allreduce_rmsnorm(xs, res, w, 1e-6)
    for m in ox.MUTANTS:
        caught = []
        for fam, W, T, H in MUTANT_CASES:
            c = sa.make_case(fam, W, T, H, seed=2, eps=1e-5)
            r, y = ox.emulate(*_case_args(c), mutant=m)
            if not ox.check(r, y, *_case_args(c))["ok"]:
                caught.append(fam)
        r, y = ox.emulate(xs, res, w, 1e-6, mutant=m)
        old = ox.old_check(r, y, rr, ry)
        rows.append((m, caught, old))
        assert caught, f"{m} passes every exact case"
    print("\nmutant          caught by (exact check)                  old 0.1 check")
    for m, caught, old in rows:
        print(f"{m:15s} {','.join(caught):40s} {'passes' if old else 'fails'}")
    old_pass = {m for m, _, old in rows if old}
    assert {"bf16_sum", "unrounded_norm", "no_eps", "gamma_first"} <= old_pass


def test_protocol_choice_and_flags_sequence():
    # one-shot only when asked for, when [T][W][H] fits the buffer and stays within 2 MiB
    assert ox.ll_protocol(8, 4, 4096, 1 << 22, 0) == (True, 8 * 4 * 8192)
    assert ox.ll_protocol(8, 4, 4096, 1 << 22, 1) == (False, 2 * 4 * 8192 + 8 * 8192)
    assert ox.ll_protocol(8, 4, 4096, 8 * 4 * 8192 - 16, 0)[0] is False
    assert ox.ll_protocol(65, 4, 4096, 1 << 24, 0) == (False, 17 * 4 * 8192 + 65 * 8192)
    f = [0, 2, 1 << 20, 0, 0, 0, 0, 0, 0]
    want = [([1, 0, 1 << 20, 0, 8192, 0, 0, 0, 0], (2, 0)),       # T=1 W=1 one-shot
            ([2, 1, 1 << 20, 0, 2 * 8192 * 3, 0, 0, 0, 0], (0, 8192)),
            ([0, 2, 1 << 20, 0, 4 * 8192, 0, 0, 0, 0], (1, 2 * 8192 * 3))]
    for (T, proto), (wf, wclear) in zip([(1, 0), (3, 1), (4, 0)], want):
        f, clear = ox.ll_flags_after(f, T, 1, 4096, proto)
        assert (f, clear) == (wf, wclear)


@pytest.mark.parametrize("W,T,one_shot", [(2, 1, True), (2, 7, False), (4, 7, True), (4, 9, False),
                                          (3, 5, False)])
def test_prefill_is_what_the_peers_deliver(W, T, one_shot):
    """Every rank's launch, replayed in Python, writes into rank p's buffer exactly the rows the
    pre-fill of p's simulated-peer launch holds, no slot is written twice, and no 16-byte vector
    of a pre-filled buffer is the sentinel."""
    H = 16
    c = sa.make_case("lamport", W, T, H, seed=3)
    sums = None if one_shot else ox.to_bf16(ox.emulate_sum(c["xs"]))
    words = (2 * ox.ceil_div(T, W) * W + T * W) * H // 2
    for p in range(W):
        delivered = np.full(words, sa.SENTINEL, np.int32)
        for r in range(W):
            if r == p:
                continue
            img = ox.ll_peer_images(T, W, H, r, one_shot, c["xs"][r], sums, words)[p]
            wrote = img != sa.SENTINEL
            assert not (wrote & (delivered != sa.SENTINEL)).any()
            delivered[wrote] = img[wrote]
        pre = ox.ll_prefill(T, W, H, p, one_shot, c["xs"], sums, words, sa.POISON)
        assert not (pre == sa.SENTINEL).any()
        got = delivered != sa.SENTINEL
        assert np.array_equal(pre[got], delivered[got])
        assert (pre[~got] == sa.POISON).all()


def test_signature_spells_out_the_ranks():
    c = sa.make_case("signature", 8, 3, 64, seed=4)
    r, _ = ox.reference(*_case_args(c))
    signs = np.stack([np.sign(ox.f64(x)) for x in c["xs"]])
    back = ((r + 255) / 2).astype(np.int64)
    for k in range(8):
        assert np.array_equal((back >> k) & 1, (signs[k] > 0).astype(np.int64))


@pytest.mark.parametrize("W,n,H", [(2, 128, 5120), (4, 77, 7168), (8, 256, 8192)])
def test_gathered_rows_graded_without_out_residual(W, n, H):
    """Rows another rank normalised are graded without its out_residual: the kernel's rank-order
    arithmetic passes (rows with an ambiguous r get the widened set), and a shifted slice, a dropped
    rank or gamma applied before rounding fail."""
    xs, res, w, _ = oa.make_inputs(W, n, H)
    xs, res = [x[:n] for x in xs], res[:n]
    _, y = ox.emulate(xs, res, w, 1e-6)
    c = ox.check(None, y, xs, res, w, 1e-6)
    print(f"\nW{W} n{n} H{H}: ambiguous r {c['amb_res']}, widened rows {c['widened_rows']}")
    assert c["ok"], ox.summary(f"gathered W{W}", c)
    assert (c["widened_rows"] > 0) == (c["amb_res"] > 0)
    for m in ("row_shift", "drop_rank", "gamma_first"):
        _, y = ox.emulate(xs, res, w, 1e-6, mutant=m)
        assert not ox.check(None, y, xs, res, w, 1e-6)["ok"], m
