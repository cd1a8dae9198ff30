"""The fused AllReduce + residual + RMSNorm kernels against the exact reference
(oracle.allreduce_exact) on ONE GPU, without processes or NCCL:

  * W = 1 through the public ops and the C entries: every block shape of both dispatch tables, every
    input family at eps 1e-6 and 1e-5, T from 1 to 129 everywhere and 4096 at H 256 (all rows
    graded) and at the widest shapes (a row sample graded); outputs written into NaN-filled buffers
    with guard rows; small grids so that blocks loop over rows.
  * The Lamport (low-latency) state across calls on one workspace, and under CUDA-graph replay.
  * The P2P transports with simulated peers: W ranks' buffers on one device, launched one rank at a
    time, with every word a launch can wait on filled beforehand so that no wait can block
    (synth.allreduce: signal-pad epochs at 2^30, Lamport slots holding the peers' rows and a
    finite poison elsewhere).
  * Argument rejections.
Each graded call prints one `EXACT <tag> ...` line (visible with -s); each test ends with the
ambiguous-element counts per family.
"""
from collections import defaultdict

import numpy as np
import pytest
import torch

from oracle import allreduce_exact as ox
from synth import allreduce as sa

pytestmark = pytest.mark.gpu
GUARD = 2


def _grade(tag, out_res, out, c, kernel, totals=None, fam=None):
    res = ox.check(out_res, out, c["xs"], c["residual"], c["weight"], c["eps"], kernel=kernel)
    print(ox.summary(tag, res))
    if totals is not None:
        t = totals[fam]
        t[0] += res["amb_res"]
        t[1] += res["amb_out"]
        t[2] += 1
    assert res["ok"], ox.summary(tag, res)
    if fam in ("exact", "signature"):
        assert res["amb_res"] == 0, "order-independent sums must be bit-exact"
    return res


def _print_totals(name, totals):
    for fam, (ar, ay, n) in sorted(totals.items()):
        print(f"EXACT-TOTAL {name} family={fam} calls={n} ambiguous(res,out)={ar},{ay}")


def _guards_untouched(buf):
    b = buf.float()
    assert torch.isnan(b[:GUARD]).all() and torch.isnan(b[-GUARD:]).all(), "guard row written"
    return buf[GUARD:-GUARD]


def _cuda(c):
    return ([x.cuda() for x in c["xs"]], c["residual"].cuda(), c["weight"].cuda())


def _ht_public(hpc, c, blocks):
    xs, res, w = _cuda(c)
    T, H = res.shape
    out, ores = sa.nan_rows(T, H, GUARD), sa.nan_rows(T, H, GUARD)
    sig = torch.zeros(1, dtype=torch.int64, device="cuda")
    o, r = out[GUARD:GUARD + T], ores[GUARD:GUARD + T]
    hpc.fuse_allreduce_rmsnorm_high_throughput(xs[0], xs[0], res, w, c["eps"], sig, 0, 1, blocks,
                                               output_x=o, output_multicast_x=o, output_residual=r)
    torch.cuda.synchronize()
    return _guards_untouched(ores).cpu(), _guards_untouched(out).cpu()


def _ll_ws(T, H, big, W=1):
    buf = sa.ll_buf_bytes(T, W, H, big)
    ws = torch.full((3 * buf // 4,), sa.SENTINEL, dtype=torch.int32, device="cuda")
    ptrs = torch.tensor([ws.data_ptr()], dtype=torch.int64, device="cuda")
    return buf, ws, ptrs, sa.new_flags(buf)


def _ll_public(hpc, c, ws, ptrs, flags, two_shot):
    xs, res, w = _cuda(c)
    T, H = res.shape
    out, ores = sa.nan_rows(T, H, GUARD), sa.nan_rows(T, H, GUARD)
    wsb = ws.view(torch.bfloat16)
    hpc.fuse_allreduce_rmsnorm_low_latency(xs[0], wsb, ptrs, wsb, flags.view(torch.uint32), 1, 0, res, w,
                                           c["eps"], 0, output_x=out[GUARD:GUARD + T],
                                           residual_out=ores[GUARD:GUARD + T], use_two_shot=two_shot)
    torch.cuda.synchronize()
    return _guards_untouched(ores).cpu(), _guards_untouched(out).cpu()


def _w1_cases(H):
    """Every family at both eps. T = 4096 is graded in full at H 256 here; at the wide shapes
    test_w1_4096_rows_subsampled grades a sample of its rows."""
    Ts = sa.TOKENS if H == 256 else sa.TOKENS[:-1]
    for i, T in enumerate(Ts):
        for j, fam in enumerate(sa.FAMILIES):
            for k, eps in enumerate(sa.EPS):
                yield i + j + k, T, fam, sa.make_case(fam, 1, T, H, seed=i, eps=eps)


def _rows(c, idx):
    return dict(xs=[x[idx] for x in c["xs"]], residual=c["residual"][idx], weight=c["weight"],
                eps=c["eps"])


@pytest.mark.parametrize("H", sa.HIDDENS)
def test_w1_public_ops(hpc, H):
    """Every bucket of both dispatchers x T x eps x family, through the public ops at W = 1."""
    totals = defaultdict(lambda: [0, 0, 0])
    for k, T, fam, c in _w1_cases(H):
        tag = f"W1 H{H} T{T} {fam} eps{c['eps']:g}"
        r, y = _ht_public(hpc, c, blocks=[1, 148][k % 2])
        _grade(f"ht {tag} shape={ox.shape_of(H, 'ht')}", r, y, c, "ht", totals, fam)
        two_shot = bool(k % 2)
        _, ws, ptrs, flags = _ll_ws(T, H, big=True)
        r, y = _ll_public(hpc, c, ws, ptrs, flags, two_shot)
        _grade(f"ll {tag} two_shot={two_shot} shape={ox.shape_of(H, 'll')}", r, y, c, "ll", totals, fam)
    _print_totals(f"W1 H{H}", totals)


@pytest.mark.parametrize("H", [7168, 16384, 16392])
def test_w1_4096_rows_subsampled(hpc, H):
    """T = 4096 at the 1024-thread LL shapes <1,1024>, <2,1024>, <4,1024> and the HT shapes <4,256>,
    <8,256>, <4,1024>: every row and guard checked for being written, a sample of 46 rows (every
    97th, and the first and last two) graded exactly. Grading all 4096 rows on the CPU would
    dominate the run."""
    T = 4096
    idx = sorted(set(range(0, T, 97)) | {1, T - 2, T - 1})
    for k, fam in enumerate(("random", "exact", "eps", "lamport")):
        for eps in (sa.EPS if fam == "eps" else (sa.EPS[k % 2],)):
            c = sa.make_case(fam, 1, T, H, seed=60 + k, eps=eps)
            sub = _rows(c, idx)
            tag = f"W1 H{H} T{T} rows={len(idx)} {fam} eps{eps:g}"
            r, y = _ht_public(hpc, c, blocks=[16, 148][k % 2])
            assert torch.isfinite(r.float()).all() and torch.isfinite(y.float()).all()
            _grade(f"ht {tag}", r[idx], y[idx], sub, "ht", fam=fam)
            _, ws, ptrs, flags = _ll_ws(T, H, big=False)
            r, y = _ll_public(hpc, c, ws, ptrs, flags, two_shot=bool(k % 2))
            assert torch.isfinite(r.float()).all() and torch.isfinite(y.float()).all()
            _grade(f"ll {tag} two_shot={bool(k % 2)}", r[idx], y[idx], sub, "ll", fam=fam)
            del ws


@pytest.mark.parametrize("H", sa.HIDDENS)
def test_w1_c_entries_small_grid(hpc, H):
    """num_max_blocks = 1 through the C entries: a block loops over several rows (the s_red[it & 1]
    double buffer), which the public LL op (one block per token) never does."""
    T = 129 if H <= 8200 else 33
    for fam in ("random", "exact", "eps"):
        c = sa.make_case(fam, 1, T, H, seed=5, eps=1e-5)
        xs, res, w = _cuda(c)
        out, ores = sa.nan_rows(T, H, GUARD), sa.nan_rows(T, H, GUARD)
        sa.ht_c(xs[0], res, w, c["eps"], out[GUARD:], ores[GUARD:], 1)
        torch.cuda.synchronize()
        _grade(f"ht-c W1 H{H} T{T} {fam} blocks=1", _guards_untouched(ores).cpu(),
               _guards_untouched(out).cpu(), c, "ht", fam=fam)
        for proto in (0, 1):
            buf, ws, ptrs, flags = _ll_ws(T, H, big=True)
            out, ores = sa.nan_rows(T, H, GUARD), sa.nan_rows(T, H, GUARD)
            sa.ll_c(xs[0], res, w, c["eps"], out[GUARD:], ores[GUARD:], ptrs, ws, flags, 1, 0, proto,
                    num_max_blocks=1)
            torch.cuda.synchronize()
            _grade(f"ll-c W1 H{H} T{T} {fam} protocol={proto} blocks=1", _guards_untouched(ores).cpu(),
                   _guards_untouched(out).cpu(), c, "ll", fam=fam)
            want, _ = ox.ll_flags_after(sa.new_flags(buf).tolist(), T, 1, H, proto)
            assert flags.tolist() == want


SEQ = (300, 8, 1, 257, 64, 256, 3)  # at H 4096, T <= 256 fits the 2 MiB one-shot limit


@pytest.mark.parametrize("big", [False, True])
@pytest.mark.parametrize("protocol", [0, 1])
def test_ll_state_across_calls(hpc, big, protocol):
    """One workspace, new data and a new batch size every call. After each call: exact outputs,
    buffer_flags as the model says, the previous call's buffer back to sentinel for exactly the
    bytes it recorded and unchanged beyond them, the current buffer holding exactly this call's
    rows, the third buffer untouched."""
    H = 4096
    buf, ws, ptrs, flags = _ll_ws(max(SEQ), H, big)
    words = buf // 4
    model = flags.tolist()
    for k, T in enumerate(SEQ):
        fam = sa.FAMILIES[k % len(sa.FAMILIES)]
        c = sa.make_case(fam, 1, T, H, seed=10 + k)
        before = ws.cpu().numpy().reshape(3, words)
        cur = model[0] % 3
        r, y = _ll_public(hpc, c, ws, ptrs, flags, protocol == 1)
        one_shot, _ = ox.ll_protocol(T, 1, H, buf, protocol)
        _grade(f"ll-state big={big} protocol={protocol} call={k} T{T} one_shot={one_shot} {fam}",
               r, y, c, "ll", fam=fam)
        model, (dirty, nbytes) = ox.ll_flags_after(model, T, 1, H, protocol)
        assert flags.tolist() == model
        after = ws.cpu().numpy().reshape(3, words)
        if dirty != cur:
            assert (after[dirty, :nbytes // 4] == sa.SENTINEL).all()
            assert np.array_equal(after[dirty, nbytes // 4:], before[dirty, nbytes // 4:])
        sums = None if one_shot else ox.to_bf16(ox.emulate_sum(c["xs"]))
        img = ox.ll_peer_images(T, 1, H, 0, one_shot, c["xs"][0], sums, words, peers=[0])[0]
        want = np.where(img != sa.SENTINEL, img, before[cur])
        assert np.array_equal(after[cur], want)
        other = 3 - cur - dirty if dirty != cur else None
        if other is not None:
            assert np.array_equal(after[other], before[other])


def test_graph_capture_replay(hpc):
    """LL (one-shot and two-shot) and HT calls captured once and replayed on new data: bit-identical
    to eager calls, exact, and buffer_flags rotating on the device with every replay."""
    H, T_ll, T_ht = 4096, 7, 129
    buf, ws, ptrs, flags = _ll_ws(T_ll, H, big=True)
    _, ws_e, ptrs_e, flags_e = _ll_ws(T_ll, H, big=True)
    x_ll = torch.zeros(T_ll, H, dtype=torch.bfloat16, device="cuda")
    r_ll = torch.zeros_like(x_ll)
    x_ht = torch.zeros(T_ht, H, dtype=torch.bfloat16, device="cuda")
    r_ht = torch.zeros_like(x_ht)
    w = torch.zeros(H, dtype=torch.bfloat16, device="cuda")
    outs = [torch.empty_like(x_ll) for _ in range(4)] + [torch.empty_like(x_ht) for _ in range(2)]
    sig = torch.zeros(1, dtype=torch.int64, device="cuda")
    wsb, wsb_e = ws.view(torch.bfloat16), ws_e.view(torch.bfloat16)

    def calls(wsv, pt, fl, o):
        for i, two in enumerate((False, True)):
            hpc.fuse_allreduce_rmsnorm_low_latency(x_ll, wsv, pt, wsv, fl.view(torch.uint32), 1, 0, r_ll, w,
                                                   1e-6, 0, output_x=o[2 * i], residual_out=o[2 * i + 1],
                                                   use_two_shot=two)
        hpc.fuse_allreduce_rmsnorm_high_throughput(x_ht, x_ht, r_ht, w, 1e-6, sig, 0, 1, 16,
                                                   output_x=o[4], output_multicast_x=o[4],
                                                   output_residual=o[5])

    model = flags.tolist()
    calls(wsb, ptrs, flags, outs)  # warm-up, eager
    for proto in (0, 1):
        model, _ = ox.ll_flags_after(model, T_ll, 1, H, proto)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        calls(wsb, ptrs, flags, outs)
    eager = [torch.empty_like(o) for o in outs]
    model_e = flags_e.tolist()
    for it in range(3):
        c_ll = sa.make_case(sa.FAMILIES[it], 1, T_ll, H, seed=20 + it)
        c_ht = sa.make_case(sa.FAMILIES[it + 3], 1, T_ht, H, seed=30 + it)
        c_ht["weight"] = c_ll["weight"]
        x_ll.copy_(c_ll["xs"][0])
        r_ll.copy_(c_ll["residual"])
        x_ht.copy_(c_ht["xs"][0])
        r_ht.copy_(c_ht["residual"])
        w.copy_(c_ll["weight"])
        g.replay()
        calls(wsb_e, ptrs_e, flags_e, eager)
        torch.cuda.synchronize()
        for proto in (0, 1):
            model, _ = ox.ll_flags_after(model, T_ll, 1, H, proto)
            model_e, _ = ox.ll_flags_after(model_e, T_ll, 1, H, proto)
        assert flags.tolist() == model and flags_e.tolist() == model_e
        for o, e in zip(outs, eager):
            assert torch.equal(o.view(torch.int16), e.view(torch.int16))
        for i in range(2):
            _grade(f"graph replay={it} ll two_shot={bool(i)}", outs[2 * i + 1].cpu(), outs[2 * i].cpu(),
                   c_ll, "ll")
        _grade(f"graph replay={it} ht", outs[5].cpu(), outs[4].cpu(), c_ht, "ht")


HT_SIM = [(W, H) for W in (2, 3, 4, 8) for H in (8, 264, 4096, 16392)]


@pytest.mark.parametrize("W,H", HT_SIM)
def test_ht_simulated_peers(hpc, W, H):
    """The P2P high-throughput kernel (mode 2 at W = 2, mode 3 beyond) with W ranks on one device.
    Every launch: out_residual of its slice exact, the identical normalised rows in every rank's
    output buffer and nothing written elsewhere, and the signal-pad bookkeeping (epoch + 1, done
    word 0, entry 2e + 1 and exit 2e + 2 posted at slot `rank` of every pad). Then a rank with an
    empty slice: it takes part in the epochs and writes nothing."""
    per = 7
    n = per * W
    totals = defaultdict(lambda: [0, 0, 0])
    sim = None
    for rnd, fam in enumerate(("signature", "exact", "random")):
        c = sa.make_case(fam, W, n, H, seed=40 + rnd)
        if sim is None:
            sim = sa.HtSim(c["xs"], H)
        else:
            for b, x in zip(sim.ins, c["xs"]):
                b.copy_(x)
            for o in sim.outs:
                o.fill_(float("nan"))
        res, w = c["residual"].cuda(), c["weight"].cuda()
        ores = torch.full_like(res, float("nan"))
        for rank in range(W):
            s, e = rank * per, (rank + 1) * per
            pads_before = [p.cpu().clone() for p in sim.pads]
            sim.launch(rank, s, e, res[s:], w, c["eps"], ores[s:], num_max_blocks=[1, 4, 148][rnd])
            torch.cuda.synchronize()
            for p, pad in enumerate(sim.pads):
                got, want = pad.cpu(), pads_before[p].clone()
                if p == rank:
                    want[:32] = sa.ARRIVED
                    want[32], want[33] = rnd + 1, 0
                want[rank], want[16 + rank] = 2 * rnd + 1, 2 * rnd + 2
                assert torch.equal(got, want), (p, got.tolist(), want.tolist())
            for o in sim.outs:  # rows of ranks not yet launched stay NaN
                assert torch.equal(o[s:e].view(torch.int16), sim.outs[0][s:e].view(torch.int16))
                assert torch.isnan(o[e:].float()).all()
            assert torch.isnan(ores[e:].float()).all()
        out = sim.outs[0].cpu()
        for o in sim.outs:
            assert torch.equal(o.cpu().view(torch.int16), out.view(torch.int16))
        _grade(f"ht-sim W{W} H{H} T{n} {fam} mode={2 if W == 2 else 3}", ores.cpu(), out, c, "ht", totals, fam)
    # empty slice: one block joins both barriers, writes nothing
    outs_before = [o.cpu().clone() for o in sim.outs]
    ores_before = ores.cpu().clone()
    sim.launch(0, n, n, res[n:], w, c["eps"], ores[n:], num_max_blocks=4)
    torch.cuda.synchronize()
    assert int(sim.pads[0][32]) == 4 and int(sim.pads[0][33]) == 0
    assert all(int(p[0]) == 7 and int(p[16]) == 8 for p in sim.pads)
    for o, b in zip(sim.outs, outs_before):
        assert torch.equal(o.cpu().view(torch.int16), b.view(torch.int16))
    assert torch.equal(ores.cpu().view(torch.int16), ores_before.view(torch.int16))
    _print_totals(f"ht-sim W{W} H{H}", totals)


LL_SIM = [(W, proto, H, T) for W in (2, 4) for proto in (0, 1) for H in (8, 2056, 8192) for T in (1, 7, 33)]


@pytest.mark.parametrize("W,protocol,H,T", LL_SIM)
def test_ll_simulated_peers(hpc, W, protocol, H, T):
    """The Lamport kernel (one-shot and two-shot, P2P stores, no multicast) with W - 1 simulated
    peers: exact outputs for every token, and afterwards each peer's workspace holds exactly this
    rank's scattered or broadcast rows at the layout's slots and the sentinel everywhere else."""
    totals = defaultdict(lambda: [0, 0, 0])
    for rank in sorted({0, W - 1, T % W}):
        for fam in ("lamport", "exact", "signature"):
            c = sa.make_case(fam, W, T, H, seed=50 + rank)
            buf = sa.ll_buf_bytes(T, W, H, big=True)
            out, ores = sa.nan_rows(T, H, GUARD), sa.nan_rows(T, H, GUARD)
            one_shot, own, peers, flags, sums = sa.ll_sim(
                c["xs"], c["residual"], c["weight"], c["eps"], rank, protocol, buf, out[GUARD:GUARD + T],
                ores[GUARD:GUARD + T], num_max_blocks=(0 if T != 7 else 1))
            torch.cuda.synchronize()
            _grade(f"ll-sim W{W} rank{rank} protocol={protocol} one_shot={one_shot} H{H} T{T} {fam}",
                   _guards_untouched(ores).cpu(), _guards_untouched(out).cpu(), c, "ll", totals, fam)
            words = buf // 4
            want = ox.ll_peer_images(T, W, H, rank, one_shot, c["xs"][rank], sums, words)
            for p, ws in peers.items():
                got = ws.cpu().numpy().reshape(3, words)
                assert np.array_equal(got[1], want[p]), f"peer {p} image"
                assert (got[0] == sa.SENTINEL).all() and (got[2] == sa.SENTINEL).all()
            o = own.cpu().numpy().reshape(3, words)
            assert (o[0] == sa.SENTINEL).all() and (o[2] == sa.SENTINEL).all()
            _, used = ox.ll_protocol(T, W, H, buf, protocol)
            assert flags.tolist() == [2, 1, buf, 0, used, 0, 0, 0, 0]
    _print_totals(f"ll-sim W{W} protocol={protocol} H{H} T{T}", totals)


@pytest.mark.parametrize("what", ["hidden_not_multiple_of_8", "hidden_too_large", "world_too_large",
                                  "rank_negative", "rank_past_world"])
def test_rejections_before_launch(hpc, what):
    H = {"hidden_not_multiple_of_8": 12, "hidden_too_large": 32776}.get(what, 64)
    world = 17 if what == "world_too_large" else 2
    rank = {"rank_negative": -1, "rank_past_world": 2}.get(what, 0)
    x = torch.ones(1, H, dtype=torch.bfloat16, device="cuda")
    w = torch.ones(H, dtype=torch.bfloat16, device="cuda")
    out, ores = sa.nan_rows(1, H, 0), sa.nan_rows(1, H, 0)
    sig = torch.zeros(world, dtype=torch.int64, device="cuda")
    peers = ([x.data_ptr()] * world, [out.data_ptr()] * world)
    with pytest.raises(RuntimeError):
        sa.ht_c(x, x, w, 1e-6, out, ores, 1, sig, peers, rank, world)
    ws = torch.full((1024,), sa.SENTINEL, dtype=torch.int32, device="cuda")
    ptrs = torch.full((world,), ws.data_ptr(), dtype=torch.int64, device="cuda")
    flags = sa.new_flags(1024)
    with pytest.raises(RuntimeError):
        sa.ll_c(x, x, w, 1e-6, out, ores, ptrs, ws, flags, world, rank, 0)
    torch.cuda.synchronize()
    assert torch.isnan(out.float()).all() and torch.isnan(ores.float()).all()
    assert flags.tolist() == sa.new_flags(1024).tolist()
    assert (ws == sa.SENTINEL).all()
