"""Fused speculative sampler on the GPU against the numpy oracle: tokens and counts equal exactly on
inputs whose decisions clear the rounding margins (synth/spec_sampler.py); recovered and bonus
tokens equal hpc.fused_sampler on the same rows; the internal Philox noise reproduced from its
launch offset and its law; CUDA-graph replay; concurrent streams; argument checks."""
import numpy as np
import pytest
import torch

from oracle import sampler as osm, spec_sampler as osp
from synth import spec_sampler as ssp
from test_spec_sampler_cpu import law_check, law_inputs

pytestmark = pytest.mark.gpu


def _dev(x):
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _temp(t):
    return _dev(t) if isinstance(t, np.ndarray) else float(t)


def _call(hpc, case, internal=False, seed=0):
    n = case["np"]
    logits = case["store_t"].cuda()[:, :n["V"]]
    return hpc.fused_speculative_sampler(
        logits, _dev(n["draft_token_ids"]), draft_probs=_dev(n["draft_probs"]),
        temperature=_temp(n["temperature"]), uniform=None if internal else _dev(n["uniform"]),
        gumbel_noise=None if internal else _dev(n["noise"]), seed=seed)


def _oracle(case, uniform=None, noise=None):
    n = case["np"]
    return osp.spec_sample(n["store"], n["V"], n["draft_token_ids"], draft_probs=n["draft_probs"],
                           temperature=n["temperature"],
                           uniform=n["uniform"] if uniform is None else uniform,
                           noise=n["noise"] if noise is None else noise)


@pytest.mark.parametrize("dt,B,K,V,probs,forms", ssp.GRID)
def test_matches_oracle(hpc, dt, B, K, V, probs, forms):
    case = ssp.case(dt, B, K, V, probs, forms)
    out, nacc = _call(hpc, case)
    want, want_n = _oracle(case)
    assert out.shape == (B, K + 1) and out.dtype == torch.int32 and nacc.dtype == torch.int32
    bad = np.nonzero((out.cpu().numpy() != want).any(1) | (nacc.cpu().numpy() != want_n))[0]
    assert bad.size == 0, (bad[:8], out.cpu().numpy()[bad[:4]], want[bad[:4]])


@pytest.mark.parametrize("dt,V", [("fp32", 4096), ("bf16", 151936)])
def test_recovered_and_bonus_equal_fused_sampler(hpc, dt, V):
    """One-hot drafts: the token at position num_accepted is fused_sampler's on that row with the
    same noise, the rejected draft excluded (no draft for the bonus)."""
    case = ssp.make_case(11, 32, 3, V, torch.float32 if dt == "fp32" else torch.bfloat16, pad=128)
    n = case["np"]
    out, nacc = _call(hpc, case)
    out, nacc = out.cpu().numpy(), nacc.cpu().numpy()
    t = n["temperature"]
    K = 3
    sampling = np.nonzero(t > 0)[0]
    rows = sampling * (K + 1) + nacc[sampling]
    drafts = np.array([n["draft_token_ids"][b, nacc[b]] if nacc[b] < K else -1 for b in sampling], np.int64)
    logits = case["store_t"].cuda()[:, :V][torch.from_numpy(rows).cuda()]
    ref = hpc.fused_sampler(logits, temperature=_dev(t[sampling]), gumbel_noise=_dev(n["noise"][rows]),
                            draft_token_ids=_dev(drafts))
    assert sampling.size >= 8
    assert np.array_equal(ref.cpu().numpy()[:, 0], out[sampling, nacc[sampling]])


def test_internal_noise_matches_philox_oracle(hpc):
    B, K, V, seed = 64, 3, 120832, 4321
    for probs in (False, True):
        case = ssp.make_case(21 + probs, B, K, V, torch.bfloat16, probs=probs)
        off = hpc.sampler._rng_offset()
        out, nacc = _call(hpc, case, internal=True, seed=seed)
        assert hpc.sampler._rng_offset() == off + 1
        g = osm.philox_gumbel(seed, off, B * (K + 1), V)
        u = osp.philox_uniforms(seed, off, B, K)
        want, want_n = _oracle(case, u, g)
        n = case["np"]
        kw = dict(draft_probs=n["draft_probs"], temperature=n["temperature"], uniform=u)
        ok = np.array([ssp.request_ok(n["store"], V, n["draft_token_ids"], kw, g, b) for b in range(B)])
        assert ok.mean() >= 0.9
        assert np.array_equal(out.cpu().numpy()[ok], want[ok]) and np.array_equal(nacc.cpu().numpy()[ok], want_n[ok])
    # a call with given noise consumes no offset
    off = hpc.sampler._rng_offset()
    _call(hpc, case)
    assert hpc.sampler._rng_offset() == off


@pytest.mark.parametrize("kind", ["onehot", "probs", "fallback"])
def test_internal_noise_law(hpc, kind):
    inp = law_inputs(kind, {"onehot": 11, "probs": 12, "fallback": 13}[kind])
    out, nacc = hpc.fused_speculative_sampler(
        _dev(inp["store"]), _dev(inp["draft"]), draft_probs=_dev(inp["q"]), temperature=float(inp["t"]),
        seed=97)
    law_check(out.cpu().numpy()[:, 0], nacc.cpu().numpy(), inp, kind)


def test_graph_replay(hpc):
    case = ssp.make_case(31, 16, 2, 4096, torch.bfloat16, probs=True)
    n = case["np"]
    eager = _call(hpc, case)
    logits = case["store_t"].cuda()[:, :4096]
    args = (_dev(n["draft_token_ids"]), _dev(n["draft_probs"]), _dev(n["temperature"]),
            _dev(n["uniform"]), _dev(n["noise"]))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        hpc.fused_speculative_sampler(logits, args[0], draft_probs=args[1], temperature=args[2],
                                      uniform=args[3], gumbel_noise=args[4])
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        given = hpc.fused_speculative_sampler(logits, args[0], draft_probs=args[1], temperature=args[2],
                                              uniform=args[3], gumbel_noise=args[4])
        own = hpc.fused_speculative_sampler(logits, args[0], draft_probs=args[1], temperature=args[2],
                                            seed=5)
    draws = []
    for _ in range(20):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(given[0], eager[0]) and torch.equal(given[1], eager[1])
        draws.append(own[0].clone())
    assert len({tuple(d.cpu().numpy().ravel()) for d in draws}) > 10


def test_concurrent_streams_match_eager(hpc):
    cases = [ssp.make_case(400 + i, 16, 1 + i % 4, 120832, torch.bfloat16, probs=bool(i % 2)) for i in range(8)]
    ref = [_call(hpc, c) for c in cases]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in cases]
    outs = []
    for c, s in zip(cases, streams):
        with torch.cuda.stream(s):
            outs.append(_call(hpc, c))
    torch.cuda.synchronize()
    for (o, n), (r, rn) in zip(outs, ref):
        assert torch.equal(o, r) and torch.equal(n, rn)


def test_nan_greedy_row_emits_id_zero(hpc):
    x = torch.randn(4, 4096, device="cuda")
    x[0] = float("nan")  # request 0, position 0: no non-NaN logit, so a_0 = 0
    x[2, 17] = 50.0
    d = torch.tensor([[0], [5]], dtype=torch.int32, device="cuda")
    out, n = hpc.fused_speculative_sampler(x, d)
    a1 = int(x[1].argmax())
    assert out[0].cpu().tolist() == [0, a1] and n[0].item() == 1
    assert out[1].cpu().tolist() == [17, -1] and n[1].item() == 0


def test_validation_raises(hpc):
    x = torch.randn(8, 4096, device="cuda")
    d = torch.zeros(4, 1, dtype=torch.int64, device="cuda")
    u = torch.rand(4, 1, device="cuda")
    g = torch.zeros(8, 4096, device="cuda")
    bad = [
        (x, torch.zeros(4, 1, dtype=torch.int16, device="cuda"), dict(seed=1)),
        (x, torch.zeros(8, 0, dtype=torch.int64, device="cuda"), dict(seed=1)),
        (torch.randn(18, 4096, device="cuda"), torch.zeros(2, 9, dtype=torch.int64, device="cuda"), dict(seed=1)),
        (x, torch.zeros(3, 1, dtype=torch.int64, device="cuda"), dict(seed=1)),
        (x, d, dict(temperature=0.7)),  # own noise without a seed
        (x, d, dict(temperature=torch.ones(4, device="cuda"), seed=0)),
        (x, d, dict(temperature=0.7, uniform=u)),
        (x, d, dict(temperature=0.7, gumbel_noise=g)),
        (x, d, dict(temperature=0.7, uniform=u, gumbel_noise=g[:4])),
        (x, d, dict(temperature=0.7, draft_probs=torch.zeros(4, 1, 4095, device="cuda"), seed=1)),
        (x, d, dict(temperature=torch.ones(3, device="cuda"), seed=1)),
        (torch.randn(8, 4100, device="cuda"), d, dict(seed=1)),
        (torch.randn(8, 4096 + 2, device="cuda")[:, :4096], d, dict(seed=1)),
        (torch.randn(8, 4096, device="cuda").half(), d, dict(seed=1)),
    ]
    for logits, drafts, kw in bad:
        with pytest.raises((RuntimeError, ValueError)):
            hpc.fused_speculative_sampler(logits, drafts, **kw)
    out, n = hpc.fused_speculative_sampler(x, d)  # greedy needs no seed
    assert out.shape == (4, 2) and n.shape == (4,)
