"""MLA prefill (hpc.attention_prefill_mla_bf16, csrc/prefill_mla.cu) against the exact fp64
reference of oracle/prefill_mla.py: element-wise bound and aggregate check over head counts, Q-tile
edges, prefixes, ragged batches with empty and key-short requests, a 32k-token request, strided
views and a given output, repeatability, and CUDA-graph replay (one graph on new contents and new
lengths, two graphs concurrently on two streams)."""
import math

import pytest
import torch

from oracle import prefill_mla as om
from synth import prefill_mla as sm

pytestmark = pytest.mark.gpu

Q_EDGES = [1, 127, 128, 129, 255]
PREFIXES = [0, 1, 63, 128, 0]


def _dev(d):
    """The case on the GPU, with k_nope / v / k_pe as views of the kv and latent buffers."""
    g = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in d.items()
         if k not in ("k_nope", "v", "k_pe")}
    g.update(k_nope=g["kv"][..., :128], v=g["kv"][..., 128:], k_pe=g["latent"][:, 512:])
    return g


def _run(hpc, d, **kw):
    g = _dev(d)
    y = hpc.attention_prefill_mla_bf16(g["q"], g["k_nope"], g["k_pe"], g["v"], g["cu_seqlens_q"],
                                       g["cu_seqlens_kv"], d["max_q"], d["scale"], **kw)
    torch.cuda.synchronize()
    return y


def _check(y, d, tag, rows=None):
    r = om.check(y.float().cpu(), d, rows=rows, device="cuda")
    print(f"EXACT mla_prefill {tag} worst={r['worst']:.3f} rel={r['rel']:.3g} "
          f"oracle_rel={r['rel_oracle']:.3g}")
    assert r["nan_ok"] and r["ok_a"] and r["ok_b"], (tag, r)
    return r


@pytest.mark.parametrize("h", [1, 8, 16, 32, 64, 128])
def test_mla_prefill_heads_tile_edges(hpc, h):
    kv = [q + p for q, p in zip(Q_EDGES, PREFIXES)]
    for i, kind in enumerate(sm.KINDS):
        d = sm.make_case(Q_EDGES, kv, h, seed=10 * h + i, kind=kind)
        _check(_run(hpc, d), d, f"h{h} {kind}")


@pytest.mark.parametrize("kind", sm.KINDS)
def test_mla_prefill_long_prefix(hpc, kind):
    d = sm.make_case([4097, 129], [4097 + 3000, 129 + 1], 8, seed=3, kind=kind, extra_q=100)
    _check(_run(hpc, d), d, f"4097 over 3000 {kind}")


def test_mla_prefill_ragged_empty_and_short_keys(hpc):
    # empty requests (no queries, with and without keys) and one request with 50 more queries
    # than keys: its first 50 rows see no key and must be zeros
    q_lens, kv_lens = [0, 200, 0, 300, 5, 0], [10, 200, 0, 250, 5, 0]
    for i, kind in enumerate(sm.KINDS):
        d = sm.make_case(q_lens, kv_lens, 16, seed=40 + i, kind=kind)
        y = _run(hpc, d)
        assert (y[200:250] == 0).all()
        _check(y, d, f"ragged {kind}")


def test_mla_prefill_32k(hpc):
    n = 32768
    d = sm.make_case([n], [n], 16, seed=5)
    rows = torch.zeros(n, dtype=torch.bool)
    rows[:256] = rows[-512:] = True
    rows[torch.randperm(n, generator=torch.Generator().manual_seed(1))[:1024]] = True
    _check(_run(hpc, d), d, "32k", rows=rows)


def test_mla_prefill_strided_views_and_output(hpc):
    d = sm.make_case([300, 129], [500, 129], 8, seed=7, kind="edge")
    g = _dev(d)
    tq = d["q"].size(0)
    qbuf = torch.full((tq, 8 * 192 + 64), math.nan, dtype=torch.bfloat16, device="cuda")
    qbuf[:, :8 * 192] = g["q"].reshape(tq, -1)
    q = qbuf[:, :8 * 192].view(tq, 8, 192)
    # k_nope head-major ([H, T, 128] storage: heads further apart than tokens), v token-major
    kn = g["k_nope"].transpose(0, 1).contiguous().transpose(0, 1)
    assert kn.stride(1) > kn.stride(0) and q.stride(0) == 8 * 192 + 64
    out = torch.full((tq, 8, 128), math.nan, dtype=torch.bfloat16, device="cuda")
    y = hpc.attention_prefill_mla_bf16(q, kn, g["k_pe"], g["v"], g["cu_seqlens_q"],
                                       g["cu_seqlens_kv"], d["max_q"], d["scale"], output=out)
    torch.cuda.synchronize()
    assert y.data_ptr() == out.data_ptr()
    _check(y, d, "strided")


def test_mla_prefill_repeatable_bits(hpc):
    d = sm.make_case([3000, 17, 700], [5000, 17, 700], 32, seed=8)
    a, b = _run(hpc, d), _run(hpc, d)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


class _Static:
    """Fixed-size device buffers a graph is captured on; load() puts a case into them."""

    def __init__(self, tq, tkv, h, nb):
        self.q = torch.zeros(tq, h, 192, dtype=torch.bfloat16, device="cuda")
        self.kv = torch.zeros(tkv, h, 256, dtype=torch.bfloat16, device="cuda")
        self.lat = torch.zeros(tkv, 576, dtype=torch.bfloat16, device="cuda")
        self.cq = torch.zeros(nb + 1, dtype=torch.int32, device="cuda")
        self.ck = torch.zeros(nb + 1, dtype=torch.int32, device="cuda")

    def load(self, d):
        self.q.zero_()
        self.kv.zero_()
        self.lat.zero_()
        self.q[:d["q"].size(0)] = d["q"].cuda()
        self.kv[:d["kv"].size(0)] = d["kv"].cuda()
        self.lat[:d["latent"].size(0)] = d["latent"].cuda()
        self.cq.copy_(d["cu_seqlens_q"].cuda())
        self.ck.copy_(d["cu_seqlens_kv"].cuda())

    def call(self, hpc, max_q, scale):
        return hpc.attention_prefill_mla_bf16(self.q, self.kv[..., :128], self.lat[:, 512:],
                                              self.kv[..., 128:], self.cq, self.ck, max_q, scale)

    def graded(self, y, d):
        return y[:d["q"].size(0)]


def _capture(hpc, st, max_q, scale):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        st.call(hpc, max_q, scale)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = st.call(hpc, max_q, scale)
    return g, y


def test_mla_prefill_graph_replay_new_lengths(hpc):
    d1 = sm.make_case([900, 70, 300], [900, 1000, 300], 16, seed=21)
    d2 = sm.make_case([130, 1000, 2], [1500, 1000, 2], 16, seed=22, kind="edge")
    st = _Static(1300, 2600, 16, 3)
    st.load(d1)
    g, y = _capture(hpc, st, 1000, d1["scale"])
    for d, tag in ((d1, "graph 1"), (d2, "graph 2"), (d1, "graph 1 again")):
        st.load(d)
        g.replay()
        torch.cuda.synchronize()
        _check(st.graded(y, d), d, tag)


def test_mla_prefill_two_graphs_two_streams(hpc):
    da = sm.make_case([2000, 300], [2500, 300], 32, seed=31)
    db = sm.make_case([100, 1500, 64], [100, 1600, 64], 32, seed=32, kind="pe")
    sa, sb = _Static(2300, 2805, 32, 2), _Static(1664, 1769, 32, 3)
    sa.load(da)
    sb.load(db)
    ga, ya = _capture(hpc, sa, 2000, da["scale"])
    gb, yb = _capture(hpc, sb, 1500, db["scale"])
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(torch.cuda.current_stream())
    s2.wait_stream(torch.cuda.current_stream())
    for _ in range(3):
        with torch.cuda.stream(s1):
            ga.replay()
        with torch.cuda.stream(s2):
            gb.replay()
    torch.cuda.synchronize()
    _check(sa.graded(ya, da), da, "stream a")
    _check(sb.graded(yb, db), db, "stream b")


def test_mla_prefill_rejections(hpc):
    d = _dev(sm.make_case([5, 3], [9, 3], 2, seed=1))
    f = hpc.attention_prefill_mla_bf16
    a = (d["q"], d["k_nope"], d["k_pe"], d["v"], d["cu_seqlens_q"], d["cu_seqlens_kv"])
    f(*a, 5, d["scale"])
    lat = torch.zeros(d["k_pe"].size(0), 580, dtype=torch.bfloat16, device="cuda")
    bad = [
        lambda: f(*a, 5, 0.0),
        lambda: f(*a, 5, math.nan),
        lambda: f(d["q"], d["k_nope"], lat[:, 512:576], *a[3:], 5, d["scale"]),  # 580-wide rows
        lambda: f(d["q"], d["k_nope"], d["k_pe"].cpu(), *a[3:], 5, d["scale"]),
        lambda: f(*a, 5, d["scale"], output=torch.zeros(8, 2, 128, device="cuda")),
        lambda: f(*a, 5, d["scale"],
                  output=torch.zeros(8, 2, 256, dtype=torch.bfloat16, device="cuda")[..., :128]),
    ]
    for i, call in enumerate(bad):
        with pytest.raises(RuntimeError):
            call()
            torch.cuda.synchronize()
            raise AssertionError(f"case {i} was accepted")
