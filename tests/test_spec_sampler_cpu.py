"""Fused speculative sampler without a GPU: the oracle against a vLLM-style torch chain, the law of
the emitted token (chi-square) and the acceptance rate, the planted cases and margins of the GPU
test's inputs, simulated kernel bugs that the GPU test's check must reject, the Philox uniforms,
the fake registration and the launcher's argument checks."""
import ctypes

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import sampler as osm, spec_sampler as osp
from synth import spec_sampler as ssp

# The GPU test's own cases (synth.spec_sampler.GRID) up to B (K + 1) V = 10 M logits; the larger
# ones are left out only to keep the CPU suite short.
CASES = [c for c in ssp.GRID if c[1] * (c[2] + 1) * c[3] <= 10_000_000]


def _run(case, mutations=()):
    n = case["np"]
    return osp.spec_sample(n["store"], n["V"], n["draft_token_ids"], draft_probs=n["draft_probs"],
                           temperature=n["temperature"], uniform=n["uniform"], noise=n["noise"],
                           mutations=mutations)


@pytest.fixture(scope="module")
def cases():
    # building a case redraws u and noise until every request clears the margins, and raises if
    # one cannot
    return [ssp.case(*c) for c in CASES]


@pytest.fixture(scope="module")
def results(cases):
    return [_run(c) for c in cases]


def test_grid_has_large_and_small_cases():
    assert len(CASES) >= 25 and any(c[3] == 151936 for c in CASES) and any(c[2] == 8 for c in CASES)


def test_oracle_matches_torch_chain(cases, results):
    for case, (out, nacc) in zip(cases, results):
        n = case["np"]
        B = out.shape[0]
        t = torch.from_numpy(np.broadcast_to(np.asarray(n["temperature"], np.float32), (B,)).copy())
        o, c = ssp.torch_chain(torch.from_numpy(np.ascontiguousarray(n["store"][:, :n["V"]])),
                               torch.from_numpy(n["draft_token_ids"]),
                               None if n["draft_probs"] is None else torch.from_numpy(n["draft_probs"]),
                               t, torch.from_numpy(n["uniform"]), torch.from_numpy(n["noise"]))
        assert np.array_equal(o.numpy(), out) and np.array_equal(c.numpy(), nacc)


def test_planted_cases_are_present(cases, results):
    """All accepted, first rejected, last rejected, out-of-range drafts, greedy ties at the draft,
    the empty-residual fallback, and greedy and sampling requests in one batch."""
    seen = set()
    for case, (out, nacc) in zip(cases, results):
        n = case["np"]
        d = n["draft_token_ids"]
        B, K = d.shape
        V = n["V"]
        t = np.broadcast_to(np.asarray(n["temperature"], np.float32), (B,))
        greedy = ~(t > 0)
        if greedy.any() and (~greedy).any():
            seen.add("mixed")
        for b in range(B):
            kind = "greedy" if greedy[b] else "sample"
            k = int(nacc[b])
            seen.add((kind, "all" if k == K else "first" if k == 0 else "last" if k == K - 1 else "mid"))
            assert (out[b, k + 1:] == -1).all() and 0 <= out[b, k] < V
            if k < K and not 0 <= d[b, k] < V:
                seen.add("out_of_range")
            if greedy[b] and k < K:
                x = n["store"][b * (K + 1) + k, :V]
                if 0 <= d[b, k] < V and x[d[b, k]] == x.max():
                    seen.add("greedy_tie_rejected")
            if not greedy[b] and k < K and n["draft_probs"] is not None:
                q = n["draft_probs"][b, k]
                xt = (n["store"][b * (K + 1) + k, :V] / np.float32(t[b])).astype(np.float32)
                if (osp._softmax64(xt[None])[0] <= q).all():
                    seen.add("fallback")
    for want in ("mixed", "out_of_range", "greedy_tie_rejected", "fallback"):
        assert want in seen, want
    for kind in ("greedy", "sample"):
        for pos in ("all", "first", "last"):
            assert (kind, pos) in seen, (kind, pos)


def test_margins_hold(cases):
    for case in cases:
        n = case["np"]
        kw = dict(draft_probs=n["draft_probs"], temperature=n["temperature"], uniform=n["uniform"])
        for b in range(n["draft_token_ids"].shape[0]):
            assert ssp.request_ok(n["store"], n["V"], n["draft_token_ids"], kw, n["noise"], b), b


@pytest.mark.parametrize("mutation", osp.MUTATIONS)
def test_inputs_expose_mutation(cases, results, mutation):
    """Each simulated bug changes a token or a count on at least one request of the GPU test's
    cases, so the GPU test's exact comparison rejects it."""
    for case, (out, nacc) in zip(cases, results):
        om, nm = _run(case, (mutation,))
        if not (np.array_equal(om, out) and np.array_equal(nm, nacc)):
            return
    pytest.fail(f"no case of the GPU grid exposes {mutation}")


def test_builder_raises_when_margins_cannot_be_met():
    V, K = 64, 1
    store = np.zeros((2, V), np.float32)
    store[:, 5] = 3.0  # one-hot draft 5 with u exactly p(5): the decision sits on the boundary
    xt = store[0]
    p = osp._softmax64(xt[None])[0]
    kw = dict(draft_probs=None, temperature=np.float32(1.0), uniform=np.array([[p[5]]], np.float32))
    with pytest.raises(ValueError, match="rounding decision"):
        ssp._clear_margins(np.random.default_rng(0), store, V, np.array([[5]]), kw,
                           np.zeros((2, V), np.float32), 0, tries=0)


# ---- the law of the emitted token ------------------------------------------------------------------
LAW_V, LAW_B = 16, 12000


def _law_logits(rng):
    x = (rng.standard_normal(LAW_V) * 1.5).astype(np.float32)
    return np.tile(x, (2 * LAW_B, 1)).astype(np.float32)


def law_inputs(kind, seed):
    """LAW_B requests with K = 1 on one logits row, t = 0.9: drafts drawn from q (one-hot: from a
    draft distribution r, q = one-hot), uniforms and noise from a seeded generator."""
    rng = np.random.default_rng(seed)
    store = _law_logits(rng)
    t = np.float32(0.9)
    p = osp._softmax64((store[:1] / t).astype(np.float32))[0]
    if kind == "onehot":
        r = rng.dirichlet(np.ones(LAW_V))
        q = None
        d = rng.choice(LAW_V, LAW_B, p=r)
    else:
        qd = rng.dirichlet(np.ones(LAW_V) * 0.7) if kind == "probs" else 2 * p  # 2p: empty residual
        q = np.tile(qd.astype(np.float32), (LAW_B, 1, 1))
        d = rng.choice(LAW_V, LAW_B, p=qd / qd.sum())
    u = rng.uniform(2.0 ** -24, 1 - 2.0 ** -24, (LAW_B, 1)).astype(np.float32)
    g = osm.gumbel_from_uniform(rng.uniform(2.0 ** -24, 1 - 2.0 ** -24, (2 * LAW_B, LAW_V)).astype(np.float32))
    return dict(store=store, draft=d[:, None].astype(np.int64), q=q, t=t, u=u, g=g, p=p)


def law_check(first, accepted, inp, kind):
    """Chi-square of the first emitted token against p, and the acceptance rate against
    sum_v q(v) min(1, p(v) / q(v)) = sum min(p, q) for a normalised q (one-hot drafts: the mean
    p(d) of the drafts drawn)."""
    p = inp["p"]
    counts = np.bincount(first, minlength=LAW_V)
    chi = stats.chisquare(counts, p * counts.sum())
    assert chi.pvalue > 1e-4, (kind, chi)
    if inp["q"] is None:
        rate = p[inp["draft"][:, 0]].mean()
    else:
        q = inp["q"][0, 0].astype(np.float64)
        rate = (q / q.sum() * np.minimum(1.0, p / q)).sum()
    se = np.sqrt(rate * (1 - rate) / LAW_B)
    assert abs(accepted.mean() - rate) < 5 * se, (kind, accepted.mean(), rate)


@pytest.mark.parametrize("kind", ["onehot", "probs", "fallback"])
def test_oracle_law(kind):
    inp = law_inputs(kind, {"onehot": 1, "probs": 2, "fallback": 3}[kind])
    out, nacc = osp.spec_sample(inp["store"], LAW_V, inp["draft"], draft_probs=inp["q"], temperature=inp["t"],
                                uniform=inp["u"], noise=inp["g"])
    if kind == "fallback":
        assert (nacc == 0).any()  # rejections happen, and every one falls back to p
    law_check(out[:, 0], nacc, inp, kind)


# ---- Philox uniforms, surface, fake registration, argument checks ---------------------------------
def test_philox_uniforms_follow_the_counter_layout():
    seed, off, B, K = 1234, (7 << 40) + 3, 3, 2
    u = osp.philox_uniforms(seed, off, B, K)
    for b in range(B):
        for i in range(K):
            bits = osm.philox4x32_10(np.array([0xFFFFFFFF, b * (K + 1) + i, off & 0xFFFFFFFF, off >> 32], np.uint32),
                                     np.array([seed, 0], np.uint32))[0]
            assert u[b, i] == osm.uniform_from_bits(bits)
    assert u.dtype == np.float32 and (u > 0).all() and (u < 1).all()


def test_exports_and_fake_shapes(hpc):
    from torch._subclasses.fake_tensor import FakeTensorMode

    assert "fused_speculative_sampler" in hpc.__all__
    with FakeTensorMode():
        x = torch.empty(5 * 4, 4096, device="cuda")
        d = torch.empty(5, 3, dtype=torch.int64, device="cuda")
        out, n = hpc.fused_speculative_sampler(x, d, temperature=0.7, seed=3)
        assert out.shape == (5, 4) and out.dtype == torch.int32
        assert n.shape == (5,) and n.dtype == torch.int32


def _buf(n, align_off=0):
    b = ctypes.create_string_buffer(n + 64)
    return b, ((ctypes.addressof(b) + 15) // 16) * 16 + align_off


def test_launcher_rejects_bad_arguments(hpc):
    lib = hpc._ffi.lib
    _keep, p = _buf(1 << 16)

    def call(B=4, K=3, V=4096, dtype=1, stride=4096, x=p, probs=None, temp=None, tval=0.7, u=None, g=None,
             seed=1, rec=p):
        return lib.hpc_fused_speculative_sampler_async(p, p, rec, x, stride, dtype, B, K, V, p, 1, probs, temp,
                                                       tval, u, g, seed, None)

    for kw, msg in ((dict(K=0), b"1 to 8"), (dict(K=9), b"1 to 8"), (dict(B=-1), b"exceeds"),
                    (dict(B=8192, K=7), b"exceeds"), (dict(V=4100, stride=4104), b"multiple of 8"),
                    (dict(V=262152, stride=262152), b"multiple of 8"), (dict(dtype=2), b"dtype"),
                    (dict(stride=4100), b"16-byte"), (dict(x=p + 4), b"16-byte"),
                    (dict(u=p), b"together"), (dict(g=p), b"together"), (dict(seed=0), b"seed"),
                    (dict(u=p, g=p + 4), b"aligned"), (dict(probs=p + 4), b"aligned"),
                    (dict(rec=None), b"scratch"), (dict(rec=p + 8), b"scratch")):
        assert call(**kw) == 1, kw
        assert msg in lib.hpc_last_error(), (kw, lib.hpc_last_error())
    assert call(B=0) == 0  # nothing to launch


def test_wrapper_requires_cuda_logits(hpc):
    with pytest.raises(RuntimeError, match="CUDA"):
        hpc.fused_speculative_sampler(torch.zeros(8, 4096), torch.zeros(4, 1, dtype=torch.int64), seed=1)
