"""GPU tests of the fused AllReduce + residual + RMSNorm (the only sharded path) across real
processes. World sizes that exceed the visible GPU count are skipped; W=1 runs on any box.
Processes are spawned like the reference's tests (tests/test_fuse_allreduce_rmsnorm_*.py).

Every rank grades its outputs with the exact checker (oracle.allreduce_exact) on three input
families: the random data of the reference tests (judged under the checker's ambiguity rule),
"exact" (order-independent fp32 sums, so out_residual must be bit-exact on every transport,
NVLS included: a switch that rounds the reduced value other than to nearest fails it) and
"signature" (rank r contributes +-2^r, so a dropped, doubled or misaddressed rank shows)."""
import math
import os
import sys
from pathlib import Path

import pytest
import torch
import torch.multiprocessing as mp

REPO = Path(__file__).resolve().parents[1]
pytestmark = pytest.mark.gpu


def _setup(rank):
    for p in (str(REPO), str(REPO / "hpc-ops_b200")):
        if p not in sys.path:
            sys.path.insert(0, p)
    torch.cuda.set_device(rank)


FAMILIES = ("random", "exact", "signature")


def _inputs(fam, world, n, hidden, seed=0):
    """(xs [n_pad, hidden] per rank, residual, weight, n_pad) of a family."""
    from oracle import allreduce as oa
    from synth import allreduce as sa

    if fam == "random":
        return oa.make_inputs(world, n, hidden, seed=10001 + seed)
    n_pad = (n + world - 1) // world * world
    c = sa.make_case(fam, world, n_pad, hidden, seed=seed)
    return c["xs"], c["residual"], c["weight"], n_pad


def _grade(fam, out_res, out, xs, residual, weight, rows, kernel):
    """Exact check of rows [a, b); '' when it passes, else the checker's summary line.
    out_res None: rows another rank normalised and broadcast (see oracle.allreduce_exact.check)."""
    from oracle import allreduce_exact as ox

    a, b = rows
    if a >= b:
        return ""
    res = ox.check(None if out_res is None else out_res[a:b], out[a:b], [x[a:b] for x in xs],
                   residual[a:b], weight, 1e-6, kernel=kernel)
    bad = not res["ok"] or (fam != "random" and res["amb_res"] > 0)
    return ox.summary(f"{fam} rows {a}:{b} widened_rows={res['widened_rows']}", res) if bad else ""


def _run_ht(rank, world, n, hidden, blocks, fam, port, q):
    try:
        _setup(rank)
        os.environ["HPC_B200_COMM_PORT"] = str(port)
        import hpc
        from oracle import allreduce as oa

        dev = torch.device("cuda", rank)
        xs, residual, weight, n_pad = _inputs(fam, world, n, hidden)
        comm = hpc.MulticastCommunicator(rank, world, rank, f"ht_{world}_{n}_{hidden}_{blocks}")
        in_x, in_hdl = hpc.empty_multimem(comm, [n_pad, hidden], dtype=torch.bfloat16, device=dev)
        out_x, out_hdl = hpc.empty_multimem(comm, [n_pad, hidden], dtype=torch.bfloat16, device=dev)
        in_x.zero_()
        in_x[:n] = xs[rank][:n].to(dev)
        out_x.fill_(float("nan"))  # every row must be written by its owner's broadcast
        residual = residual.to(dev)
        weight = weight.to(dev)
        out_res = torch.empty_like(residual)
        s, e = oa.token_slice(n_pad, world, rank)
        off = s * hidden * 2
        comm.Barrier()
        for _ in range(3):  # repeated calls exercise the barrier slot reuse
            hpc.fuse_allreduce_rmsnorm_high_throughput(
                in_x[s:e], in_hdl.get_multimem_buff((e - s, hidden), torch.bfloat16, off),
                residual[s:e], weight, 1e-6, in_hdl.signal_buffer_ptrs_dev, rank, world, blocks,
                out_x[s:e], out_hdl.get_multimem_buff((e - s, hidden), torch.bfloat16, off),
                out_res[s:e])
        torch.cuda.synchronize()
        comm.Barrier()
        # this rank's slice in full (its out_residual rows feed its norm), then every row of the
        # gathered output, most of which the other ranks' broadcasts wrote
        err = _grade(fam, out_res.cpu(), out_x.cpu(), xs, residual, weight, (s, min(e, n)), "ht")
        err += _grade(fam, None, out_x.cpu(), xs, residual, weight, (0, n), "ht")
        q.put((rank, not err, f"mc={in_hdl.has_multicast} {err}"))
    except Exception as ex:  # noqa: BLE001
        q.put((rank, False, repr(ex)[:500]))


def _run_ll(rank, world, seq, hidden, big_ws, two_shot, fam, port, q):
    """`seq`: token counts of consecutive calls on ONE workspace (varying batch sizes exercise the
    dirty-buffer bookkeeping); big_ws: workspace large enough for the one-shot layout."""
    try:
        _setup(rank)
        os.environ["HPC_B200_COMM_PORT"] = str(port)
        import hpc
        dev = torch.device("cuda", rank)
        nmax = max(seq)
        xs, residual, weight, _ = _inputs(fam, world, nmax, hidden)
        comm = hpc.MulticastCommunicator(rank, world, rank, f"ll_{world}_{nmax}_{hidden}_{big_ws}_{fam}")
        m_pad = 2 * math.ceil(nmax / world) * world * 3  # reference sizing (test :54-60)
        if big_ws:
            m_pad = max(m_pad, nmax * world * 3)
        ws, hdl = hpc.empty_multimem(comm, [m_pad, hidden], dtype=torch.bfloat16, device=dev)
        ws.view(torch.int32).fill_(-2147483648)  # 0x80000000 words
        mc = hdl.get_multimem_buff([m_pad, hidden], dtype=torch.bfloat16)
        buf_bytes = (m_pad * hidden * 2 // 3) // 16 * 16
        flags = torch.tensor([0, 2, buf_bytes, 0, 0, 0, 0, 0, 0], dtype=torch.int32, device=dev)
        weight = weight.to(dev)
        torch.cuda.synchronize()
        comm.Barrier()
        err = ""
        for it, n in enumerate(seq):
            # different data every call: a stale row from an earlier call cannot pass
            xs_i = [torch.roll(x[:nmax], it + 1, 0)[:n].contiguous() for x in xs]
            res_i = torch.roll(residual[:nmax], it + 2, 0)[:n].contiguous()
            x = xs_i[rank].to(dev).contiguous()
            r = res_i.to(dev).contiguous()
            out = torch.empty_like(x)
            out_res = torch.empty_like(r)
            hpc.fuse_allreduce_rmsnorm_low_latency(x, mc, hdl.data_buffer_ptrs_dev, ws,
                                                   flags.view(torch.uint32), world, rank, r,
                                                   weight, 1e-6, 0, out, out_res, True,
                                                   use_two_shot=two_shot)
            torch.cuda.synchronize()
            err += _grade(fam, out_res.cpu(), out.cpu(), xs_i, res_i, weight.cpu(), (0, n), "ll")
        comm.Barrier()
        q.put((rank, not err, f"mc={hdl.has_multicast} {err}"))
    except Exception as ex:  # noqa: BLE001
        q.put((rank, False, repr(ex)[:500]))


def _spawn(target, world, args):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    only = os.environ.get("HPC_B200_TEST_WORLDS")  # e.g. "4,8" on a multi-GPU lease: skip the rest
    if only and str(world) not in only.split(","):
        pytest.skip(f"world size {world} not selected by HPC_B200_TEST_WORLDS")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 21000 + (os.getpid() * 7 + hash(args) % 997) % 15000
    procs = [ctx.Process(target=target, args=(r, world, *args, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
    res = []
    while not q.empty():
        res.append(q.get())
    for p in procs:
        if p.is_alive():
            p.kill()
    assert len(res) == world, f"only {len(res)} of {world} ranks reported: {res}"
    assert all(r[1] for r in res), res


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("n,hidden,blocks", [(128, 5120, 16), (77, 7168, 78), (256, 8192, 32)])
def test_allreduce_rmsnorm_high_throughput(world, n, hidden, blocks):
    _spawn(_run_ht, world, (n, hidden, blocks, "random"))


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("n,hidden,blocks", [(77, 7168, 78)])
@pytest.mark.parametrize("fam", FAMILIES[1:])
def test_allreduce_rmsnorm_high_throughput_exact_families(world, n, hidden, blocks, fam):
    _spawn(_run_ht, world, (n, hidden, blocks, fam))


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("n,hidden", [(128, 5120), (77, 7168), (8, 8192)])
def test_allreduce_rmsnorm_low_latency(world, n, hidden):
    """reference grid (tests/test_fuse_allreduce_rmsnorm_low_latency.py:121-125), two-shot protocol,
    5 calls so that every Lamport buffer is reused."""
    _spawn(_run_ll, world, ((n,) * 5, hidden, False, True, "random"))


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("n,hidden", [(77, 7168)])
@pytest.mark.parametrize("two_shot", [True, False])
@pytest.mark.parametrize("fam", FAMILIES[1:])
def test_allreduce_rmsnorm_low_latency_exact_families(world, n, hidden, two_shot, fam):
    _spawn(_run_ll, world, ((n,) * 5, hidden, not two_shot, two_shot, fam))


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("two_shot", [True, False])
def test_allreduce_rmsnorm_low_latency_varying_batch(world, two_shot):
    """Decode batches change size every step: a call must clear what the PREVIOUS call dirtied,
    not what its own size suggests (64, 8, 8, 64 left stale rows behind in round 1)."""
    _spawn(_run_ll, world, ((64, 8, 8, 64, 1, 33, 64, 2), 8192, not two_shot, two_shot, "random"))


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("n", [1, 8, 32])
def test_allreduce_rmsnorm_low_latency_one_shot(world, n):
    """one-shot protocol (workspace sized [tokens][world][hidden] per buffer)."""
    _spawn(_run_ll, world, ((n,) * 5, 8192, True, False, "random"))


@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_allreduce_rmsnorm_c5_shape(world):
    """BASELINE config C5: 4096 tokens x hidden 8192 (the W=2 shape once showed max_abs_err 20)."""
    _spawn(_run_ht, world, (4096, 8192, 148, "random"))
