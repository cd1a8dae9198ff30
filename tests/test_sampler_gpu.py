"""Fused sampler on the GPU against the numpy oracle: tokens equal exactly and the penalty mask bit for
bit, over logits families chosen so that rounding cannot decide a token (synth/sampler.py); the
internal Philox noise reproduced from its launch offset; sampling statistics eagerly and under
CUDA-graph replay; concurrent streams; argument checks."""
import numpy as np
import pytest
import torch

from oracle import sampler as osm
from synth import sampler as ss

pytestmark = pytest.mark.gpu


def _dev(x):
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _param(v):
    return _dev(v) if isinstance(v, np.ndarray) else v


def _logits(case, V):
    return case["store_t"].cuda()[:, :V]


def _run_full(hpc, case, seed=0, internal=False):
    """One hpc.fused_sampler call on `case`, with its own noise or (internal) the kernel's."""
    n = case["np"]
    mask = _dev(n["penalty_mask"])
    out = hpc.fused_sampler(
        _logits(case, n["V"]), penalty_mask=mask, slot_id=_dev(n["slot_id"]),
        repetition_penalty=_param(n["repetition_penalty"]), temperature=_param(n["temperature"]),
        softmax_policy=n["softmax_policy"], topk=_param(n["topk"]), topp=_param(n["topp"]),
        max_topk=n["max_topk"], gumbel_noise=None if internal else _dev(n["noise"]), seed=seed)
    return out, mask


def _oracle_full(case, noise=None):
    n = case["np"]
    kw = {k: v for k, v in n.items() if k not in ("store", "V", "noise")}
    return osm.fused_sampler(n["store"], n["V"], noise=n["noise"] if noise is None else noise, **kw)


@pytest.mark.parametrize("dt,B,V,max_topk,policy,forms", ss.FULL_GRID)
def test_full_path_matches_oracle(hpc, dt, B, V, max_topk, policy, forms):
    case = ss.full_case(dt, B, V, max_topk, policy, forms)
    logits = _logits(case, V)
    before = logits.clone()
    out, mask = _run_full(hpc, case)
    tok, mask_ref = _oracle_full(case)
    assert out.shape == (B, 1) and out.dtype == torch.int32
    assert torch.equal(out.cpu()[:, 0], torch.from_numpy(tok)), (out.cpu()[:, 0] != torch.from_numpy(tok)).nonzero()
    assert torch.equal(mask.cpu(), torch.from_numpy(mask_ref))
    assert torch.equal(logits, before)


@pytest.mark.parametrize("dt,B,V,forms", ss.FAST_GRID)
def test_fast_path_matches_oracle(hpc, dt, B, V, forms):
    case = ss.fast_case(dt, B, V, forms)
    n = case["np"]
    logits = _logits(case, V)
    out = hpc.fused_sampler(logits, temperature=_param(n["temperature"]), gumbel_noise=_dev(n["noise"]),
                            draft_token_ids=_dev(n["draft_token_ids"]))
    tok = osm.temperature_sample(n["store"], V, temperature=n["temperature"], noise=n["noise"],
                                 draft_token_ids=n["draft_token_ids"])
    assert torch.equal(out.cpu()[:, 0], torch.from_numpy(tok))


def test_internal_noise_matches_philox_oracle(hpc):
    B, V, seed = 64, 120832, 1234
    case = ss.make_full_case(7, B, V, dtype=torch.bfloat16, policy=2)
    off = hpc.sampler._rng_offset()
    out, mask = _run_full(hpc, case, seed=seed, internal=True)
    g = osm.philox_gumbel(seed, off, B, V)
    tok, mask_ref = _oracle_full(case, g)
    n = case["np"]
    kw = {k: v for k, v in n.items() if k not in ("store", "V", "noise")}
    ok = np.array([ss.full_row_ok(n["store"], V, kw, g, b) for b in range(B)])
    assert ok.mean() >= 0.99
    assert np.array_equal(out.cpu().numpy()[ok, 0], tok[ok])
    assert hpc.sampler._rng_offset() == off + 1

    fast = ss.make_fast_case(8, B, V, dtype=torch.float32, draft=False)
    t = fast["np"]["temperature"]
    off = hpc.sampler._rng_offset()
    out = hpc.fused_sampler(_logits(fast, V), temperature=_dev(t), seed=seed)
    g = osm.philox_gumbel(seed, off, B, V)
    tok = osm.temperature_sample(fast["np"]["store"], V, temperature=t, noise=g)
    ok = np.array([osm.fast_row_gap(fast["np"]["store"][b, :V], t[b], g[b]) >= ss.MARGIN for b in range(B)])
    assert ok.mean() >= 0.99
    assert np.array_equal(out.cpu().numpy()[ok, 0], tok[ok])


def _peaked(rows):
    x = torch.full((rows, 4096), -30.0, device="cuda")
    x[:, 100:108] = torch.tensor([2.0, 1.6, 1.2, 1.0, 0.5, 0.2, 0.0, -0.5], device="cuda")
    return x


def _tv(tokens, x, T):
    p = torch.softmax(x[0].double().cpu() / T, 0).numpy()
    emp = np.bincount(tokens, minlength=x.shape[1]) / tokens.size
    return 0.5 * np.abs(emp - p).sum()


def test_internal_noise_statistics_eager_and_graph(hpc):
    T = 0.8
    x = _peaked(2000)
    a = hpc.fused_sampler(x, temperature=T, seed=77)
    b = hpc.fused_sampler(x, temperature=T, seed=77)
    assert not torch.equal(a, b)
    assert _tv(a.cpu().numpy()[:, 0], x, T) < 0.1
    # full path: top-k 8 keeps every token of the peak, so the law is softmax(x / T) too
    f = hpc.fused_sampler(x, temperature=T, topk=8, seed=77)
    assert _tv(f.cpu().numpy()[:, 0], x, T) < 0.1

    x10 = _peaked(10)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        hpc.fused_sampler(x10, temperature=T, seed=77)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = hpc.fused_sampler(x10, temperature=T, seed=77)
    draws = []
    for _ in range(200):
        g.replay()
        draws.append(out.clone())
    d = torch.cat(draws).cpu().numpy()[:, 0]
    assert len({tuple(t.cpu().numpy()[:, 0]) for t in draws}) > 100
    assert _tv(d, x10, T) < 0.1


def test_concurrent_streams_match_eager(hpc):
    """Eight streams at once: with given noise each matches its eager call; with the kernel's own
    noise each stream's launch offset advances by one per call and its tokens are those the numpy
    Philox gives for the offset read before the calls."""
    V, seed, calls = 120832, 99, 3
    cases = [ss.make_full_case(300 + i, 16, V, dtype=torch.bfloat16, policy=1 + i % 2) for i in range(8)]
    ref = [_run_full(hpc, c) for c in cases]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in cases]
    outs = []
    for c, s in zip(cases, streams):
        with torch.cuda.stream(s):
            outs.append(_run_full(hpc, c))
    torch.cuda.synchronize()
    for (o, m), (r, rm) in zip(outs, ref):
        assert torch.equal(o, r) and torch.equal(m, rm)

    fasts = [ss.make_fast_case(400 + i, 16, V, dtype=torch.bfloat16, draft=False) for i in range(8)]
    logits = [_logits(f, V) for f in fasts]
    temps = [_dev(f["np"]["temperature"]) for f in fasts]
    offsets = []
    for s in streams:
        with torch.cuda.stream(s):
            offsets.append(hpc.sampler._rng_offset())
    assert len(set(offsets)) == len(streams)
    torch.cuda.synchronize()
    outs = [[] for _ in streams]
    for _ in range(calls):  # interleaved: every stream has calls in flight at once
        for i, s in enumerate(streams):
            with torch.cuda.stream(s):
                outs[i].append(hpc.fused_sampler(logits[i], temperature=temps[i], seed=seed))
    torch.cuda.synchronize()
    for i, (s, f) in enumerate(zip(streams, fasts)):
        with torch.cuda.stream(s):
            assert hpc.sampler._rng_offset() == offsets[i] + calls
        n = f["np"]
        for k in range(calls):
            g = osm.philox_gumbel(seed, offsets[i] + k, 16, V)
            tok = osm.temperature_sample(n["store"], V, temperature=n["temperature"], noise=g)
            ok = np.array([osm.fast_row_gap(n["store"][b, :V], n["temperature"][b], g[b]) >= ss.MARGIN
                           for b in range(16)])
            assert np.array_equal(outs[i][k].cpu().numpy()[ok, 0], tok[ok]), (i, k)


def test_validation_raises(hpc):
    x = torch.randn(4, 4096, device="cuda")
    mask = torch.zeros(4, 512, dtype=torch.uint8, device="cuda")
    slot = torch.arange(4, dtype=torch.int32, device="cuda")
    bad = [
        dict(topp=0.9, softmax_policy=2, temperature=1.0, seed=1),  # top-p without top-k
        dict(topp=0.9, topk=20, seed=1),  # top-p with NONE
        dict(penalty_mask=mask, temperature=1.0, seed=1),
        dict(slot_id=slot, temperature=1.0, seed=1),
        dict(repetition_penalty=1.1, topk=20, seed=1),
        # 5 x 513 bytes: the write-back's 4-byte word would reach past the mask
        dict(penalty_mask=torch.zeros(5, 513, dtype=torch.uint8, device="cuda"), slot_id=slot,
             repetition_penalty=1.1, topk=20, seed=1),
        dict(max_topk=48, topk=20, seed=1),
        dict(topk=20, seed=0),  # no noise and no seed
        dict(temperature=1.0, seed=-3),
        dict(temperature=1.0, seed=1, draft_token_ids=torch.zeros(4, dtype=torch.int32, device="cuda")),
        dict(temperature=1.0, seed=1, draft_token_ids=torch.zeros(5, dtype=torch.int64, device="cuda")),
    ]
    for kw in bad:
        with pytest.raises((RuntimeError, ValueError)):
            hpc.fused_sampler(x, **kw)
    with pytest.raises(ValueError):
        hpc.fused_sampler(x, topk=20, seed=1, draft_token_ids=torch.zeros(4, dtype=torch.int64, device="cuda"))
    with pytest.raises(RuntimeError):
        hpc.fused_sampler(torch.randn(4096, 4, device="cuda").t(), temperature=1.0, seed=1)  # stride(1) != 1
    for V in (12345, 4100):
        with pytest.raises(RuntimeError):
            hpc.fused_sampler(torch.randn(2, V, device="cuda"), temperature=1.0, seed=1)
    with pytest.raises(RuntimeError):  # rows not 16-byte aligned
        hpc.fused_sampler(torch.randn(2, 4096 + 2, device="cuda")[:, :4096], temperature=1.0, seed=1)
