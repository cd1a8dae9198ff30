"""GPU parity tests for the decode-attention path (`pytest -m gpu` on an H100).

Everything goes through the product's public API (hpc.*  ->  C-ABI  ->  sm_90a kernels) and is
checked against the CPU oracle; integer outputs bit-exact, attention within the reference's
asserted tolerance (atol=0.2, reference tests/test_attention_decode_qpertoken_perhead_kvpertensor_fp8.py:260)
plus a much tighter relative-error bound of our own.
"""
import ctypes
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import attention as oa
from oracle import taskmap as otm

pytestmark = pytest.mark.gpu
G = Path(__file__).resolve().parent / "golden"


# ------------------------------------------------------------------------------------------------
# task map: CUDA scheduler bit-exact vs oracle and vs the product's CPU scheduler
# ------------------------------------------------------------------------------------------------
def _sched_ints(task_map_i32, num_batch, num_head_kv):
    ntpc1, ctas = int(task_map_i32[0]), int(task_map_i32[1])
    n = (ntpc1 * ctas + 1) * 12 + (num_batch * num_head_kv + 11) // 12 * 12
    return n


@pytest.mark.parametrize("num_batch", [1, 16, 200, 2048])
@pytest.mark.parametrize("num_seq_q", [1, 4])
@pytest.mark.parametrize("max_seq_kv", [130, 4096])
@pytest.mark.parametrize("num_head_kv", [1, 8])
def test_taskmap_cuda_bit_exact(hpc, num_batch, num_seq_q, max_seq_kv, num_head_kv):
    torch.manual_seed(41)
    mpl = 1024
    lens = torch.randint(1, max_seq_kv, (num_batch,), dtype=torch.int32, device="cuda") + num_seq_q
    ws_cpu = hpc.get_attention_decode_task_workspace(num_batch, max_seq_kv + num_seq_q, num_head_kv, mpl)
    ws_gpu = hpc.get_attention_decode_task_workspace(num_batch, max_seq_kv + num_seq_q, num_head_kv, mpl)
    hpc.assign_attention_decode_task(lens.cpu(), ws_cpu, num_head_kv, num_seq_q, True, mpl)
    hpc.assign_attention_decode_task(lens, ws_gpu, num_head_kv, num_seq_q, True, mpl)
    a = ws_cpu.view(torch.int32).cpu().numpy()
    b = ws_gpu.view(torch.int32).cpu().numpy()
    n = _sched_ints(a, num_batch, num_head_kv)
    assert np.array_equal(a[:n], b[:n])
    ctas = torch.cuda.get_device_properties(0).multi_processor_count
    o = otm.assign(lens.cpu().numpy(), ctas, num_head_kv, num_seq_q, 128, True, mpl).reshape(-1)
    # header ints 2..4 are allocator fields in the device workspace, zero in the packed host map
    assert np.array_equal(o[:2], b[:2]) and o[5] == b[5]
    assert np.array_equal(o[12:n], b[12:n])


def test_taskmap_reassign_same_workspace(hpc):
    """A workspace is reused every decode step: stale rows of a longer schedule must not leak."""
    ws = hpc.get_attention_decode_task_workspace(64, 8192, 8, 64)
    ctas = torch.cuda.get_device_properties(0).multi_processor_count
    for lens in ([8192] * 64, [100] * 64, [5000] * 3 + [7] * 61):
        t = torch.tensor(lens, dtype=torch.int32, device="cuda")
        hpc.assign_attention_decode_task(t, ws, 8, 1, True, 64)
        b = ws.view(torch.int32).cpu().numpy()
        o = otm.assign(lens, ctas, 8, 1, 128, True, 64).reshape(-1)
        n = _sched_ints(b, 64, 8)
        assert np.array_equal(o[12:n], b[12:n])


# ------------------------------------------------------------------------------------------------
# decode attention
# ------------------------------------------------------------------------------------------------
def _run_decode(hpc, d, num_batch, num_seq_q, hkv, min_process_len=1024, use_task_map=True,
                cpu_assign=False, output=None):
    lens = d["kv_lens_total"]
    task_map = None
    if use_task_map:
        task_map = hpc.get_attention_decode_task_workspace(num_batch, int(lens.max()), hkv, min_process_len)
        hpc.assign_attention_decode_task(lens.cpu() if cpu_assign else lens, task_map, hkv, num_seq_q,
                                         True, min_process_len)
    return hpc.attention_decode_fp8(
        d["q"], d["kvcache"][:, 0], d["kvcache"][:, 1], d["block_ids"], lens, d["q_scale"],
        d["k_scale"], d["v_scale"], mtp=num_seq_q - 1, new_kv_included=True,
        quant_type=hpc.QuantType.QPERTOKEN_PERHEAD_KPERTENSOR_VPERTENSOR, splitk=True,
        task_map=task_map, output=output)


def _check(my, gt, tag="", atol=0.2, rel_max=0.03):
    """Reference tolerance (atol) plus a relative-L2 bound of our own. The bound is loose enough for
    the one legitimate difference from the oracle: split-k chunks quantise P relative to the chunk
    maximum instead of the row maximum, which moves e4m3 rounding points (outputs of random V
    cancel to ~|v|/sqrt(n), so that noise is a few percent of the output norm)."""
    my = my.float().cpu()
    gt = gt.float().cpu()
    err = (my - gt).abs()
    rel = err.norm() / gt.norm().clamp_min(1e-6)
    assert torch.isfinite(my).all(), f"{tag}: non-finite output"
    assert torch.allclose(my, gt, atol=atol), f"{tag}: max abs err {err.max():.4f}"
    assert rel < rel_max, f"{tag}: relative error {rel:.4f}"


@pytest.mark.parametrize("num_batch", [1, 16, 200])
@pytest.mark.parametrize("num_seq_q", [1, 2, 3, 4])
@pytest.mark.parametrize("max_seq_kv", [1024, 4096])
@pytest.mark.parametrize("kv_head_q_head", [(1, 8), (4, 32), (8, 32)])
@pytest.mark.parametrize("layout", ["NHD", "HND"])
def test_decode_fp8_vs_oracle(hpc, num_batch, num_seq_q, max_seq_kv, kv_head_q_head, layout):
    """Parameter grid of reference tests/test_attention_decode_qpertoken_perhead_kvpertensor_fp8.py:263-273
    (+ the GQA 32/8 shape of BASELINE config C2)."""
    hkv, hq = kv_head_q_head
    if num_batch == 200 and max_seq_kv == 4096 and hkv == 8:
        pytest.skip("CPU oracle too slow for this cell; covered by the sampled full-size test")
    g = torch.Generator().manual_seed(41)
    lens = torch.randint(1, max_seq_kv, (num_batch,), generator=g, dtype=torch.int32) + num_seq_q
    d = oa.make_decode_fp8_inputs(num_batch, num_seq_q, lens, hkv, hq, seed=41, layout=layout,
                                  device="cuda")
    my = _run_decode(hpc, d, num_batch, num_seq_q, hkv)
    dc = {k: v.cpu() for k, v in d.items()}
    gt = oa.decode_fp8_kvpertensor(dc["q"], dc["kvcache"][:, 0], dc["kvcache"][:, 1], dc["block_ids"],
                                   dc["kv_lens_total"], dc["q_scale"], dc["k_scale"], dc["v_scale"],
                                   num_seq_q)
    _check(my, gt, f"B{num_batch} Sq{num_seq_q} S{max_seq_kv} {kv_head_q_head} {layout}")


@pytest.mark.parametrize("lens", [[1], [2, 64, 65, 127, 128, 129, 255, 256, 257], [4, 4, 4],
                                  [40000], [129] * 5, [131] * 37])
@pytest.mark.parametrize("num_seq_q", [1, 4])
def test_decode_fp8_edge_lengths(hpc, lens, num_seq_q):
    """Ragged / boundary lengths: single token, exact tile multiples, tails shorter than num_seq_q
    (causal window spilling into the previous chunk), one request split over every CTA."""
    lens = [max(L, num_seq_q) for L in lens]
    B = len(lens)
    d = oa.make_decode_fp8_inputs(B, num_seq_q, lens, 2, 8, seed=7, device="cuda")
    for mpl in (64, 1024):
        my = _run_decode(hpc, d, B, num_seq_q, 2, min_process_len=mpl)
        dc = {k: v.cpu() for k, v in d.items()}
        gt = oa.decode_fp8_kvpertensor(dc["q"], dc["kvcache"][:, 0], dc["kvcache"][:, 1],
                                       dc["block_ids"], dc["kv_lens_total"], dc["q_scale"],
                                       dc["k_scale"], dc["v_scale"], num_seq_q)
        _check(my, gt, f"lens {lens[:4]} Sq{num_seq_q} mpl{mpl}")


def test_decode_fp8_golden_fixtures(hpc):
    """Outputs of the reference's own test reference function (tests/golden/make_golden.py)."""
    for name in ("decode_fp8_b2_nhd.npz", "decode_fp8_b5_hnd.npz"):
        z = np.load(G / name)
        B, sq, hkv, hq, D, bs = map(int, z["meta"])
        kv = torch.from_numpy(z["kvcache"]).view(torch.float8_e4m3fn).cuda()
        if int(z["layout"][0]) == 1:
            kv = kv.permute(0, 1, 3, 2, 4).contiguous().permute(0, 1, 3, 2, 4)
        d = dict(q=torch.from_numpy(z["q"]).view(torch.float8_e4m3fn).cuda(), kvcache=kv,
                 block_ids=torch.from_numpy(z["block_ids"]).cuda(),
                 kv_lens_total=torch.from_numpy(z["kv_lens_total"]).cuda(),
                 q_scale=torch.from_numpy(z["q_scale"]).cuda(),
                 k_scale=torch.from_numpy(z["k_scale"]).cuda(),
                 v_scale=torch.from_numpy(z["v_scale"]).cuda())
        my = _run_decode(hpc, d, B, sq, hkv)
        _check(my, torch.from_numpy(z["out"]), name)


def test_decode_fp8_without_task_map_and_cpu_assigned_map(hpc):
    """Also: q as a row-strided view of a fused qkv buffer, and output as a row-strided view
    (split-k combine and the direct write of unsplit pairs): the same bits, and nothing written
    outside the output view."""
    from test_decode_bf16_gpu import _strided_output, _strided_q

    d = oa.make_decode_fp8_inputs(16, 2, [777] * 16, 4, 32, seed=5, device="cuda")
    a = _run_decode(hpc, d, 16, 2, 4, use_task_map=False)
    b = _run_decode(hpc, d, 16, 2, 4, min_process_len=512)
    c = _run_decode(hpc, d, 16, 2, 4, min_process_len=512, cpu_assign=True)
    assert torch.equal(a, b) and torch.equal(b, c)
    g = _run_decode(hpc, dict(d, q=_strided_q(d["q"], 16)), 16, 2, 4, min_process_len=512)
    assert torch.equal(a, g)
    base = _run_decode(hpc, d, 16, 2, 4, min_process_len=4096)  # some pairs split, some not
    for mpl, want in ((512, a), (4096, base)):
        buf, view = _strided_output(d["q"], 128)
        y = _run_decode(hpc, d, 16, 2, 4, min_process_len=mpl, output=view)
        assert y.data_ptr() == view.data_ptr() and torch.equal(y, want)
        assert bool((buf[:, 32 * 128:] == 7.0).all()), "written outside the output view"


def test_decode_fp8_paging_invariance_and_schedule_invariance(hpc):
    """Size-independent properties: (1) relocating pages (different block_ids, same logical KV)
    leaves the output bit-identical; (2) a different chunking (min_process_len) changes only fp32
    summation order."""
    B, hkv, hq = 8, 8, 32
    d = oa.make_decode_fp8_inputs(B, 1, [3000 + 17 * i for i in range(B)], hkv, hq, seed=11, device="cuda")
    base = _run_decode(hpc, d, B, 1, hkv, min_process_len=64)
    nblk = d["kvcache"].shape[0]
    perm = torch.randperm(nblk, device="cuda")
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(nblk, device="cuda")
    d2 = dict(d)
    d2["kvcache"] = d["kvcache"][perm]          # block j now holds old block perm[j]
    d2["block_ids"] = inv[d["block_ids"].long()].to(torch.int32)
    moved = _run_decode(hpc, d2, B, 1, hkv, min_process_len=64)
    assert torch.equal(base, moved)
    other = _run_decode(hpc, d, B, 1, hkv, min_process_len=2048)
    assert torch.allclose(base.float(), other.float(), atol=2e-2)


def test_decode_fp8_full_size_c2_sampled(hpc):
    """BASELINE config C2 (bs=64, GQA 32/8, d=128, seq=8192) at full size; the CPU oracle checks a
    sample of requests (each request's output depends only on its own KV)."""
    B, hkv, hq, S = 64, 8, 32, 8192
    d = oa.make_decode_fp8_inputs(B, 1, [S] * B, hkv, hq, seed=41, device="cuda")
    my = _run_decode(hpc, d, B, 1, hkv, min_process_len=64)
    assert torch.isfinite(my.float()).all()
    for bi in (0, 31, 63):
        sub = dict(q=d["q"][bi:bi + 1].cpu(), kvcache=d["kvcache"].cpu(),
                   block_ids=d["block_ids"][bi:bi + 1].cpu(),
                   kv_lens_total=d["kv_lens_total"][bi:bi + 1].cpu(),
                   q_scale=d["q_scale"][bi:bi + 1].cpu(), k_scale=d["k_scale"].cpu(),
                   v_scale=d["v_scale"].cpu())
        gt = oa.decode_fp8_kvpertensor(sub["q"], sub["kvcache"][:, 0], sub["kvcache"][:, 1],
                                       sub["block_ids"], sub["kv_lens_total"], sub["q_scale"],
                                       sub["k_scale"], sub["v_scale"], 1)
        _check(my[bi:bi + 1], gt, f"C2 request {bi}")


# ------------------------------------------------------------------------------------------------
# k-per-token / v-per-head variant (quant_type 0): scales in the cache allocation's extra rows
# ------------------------------------------------------------------------------------------------
def _run_decode_kpt(hpc, d, num_batch, num_seq_q, hkv, min_process_len=2048, use_task_map=True):
    tm = None
    if use_task_map:
        tm = hpc.get_attention_decode_task_workspace(num_batch, int(d["kv_lens_total"].max()), hkv,
                                                     min_process_len)
        hpc.assign_attention_decode_task(d["kv_lens_total"], tm, hkv, num_seq_q, True, min_process_len)
    return hpc.attention_decode_fp8(
        d["q"], d["kcache"], d["vcache"], d["block_ids"], d["kv_lens_total"], d["q_scale"],
        d["k_scale"], d["v_scale"], mtp=num_seq_q - 1, new_kv_included=True,
        quant_type=hpc.QuantType.QPERTOKEN_PERHEAD_KPERTOKEN_PERHEAD_VPERHEAD, task_map=tm)


def _oracle_kpt(d, num_seq_q):
    c = {k: v.cpu() for k, v in d.items()}
    return oa.decode_fp8_kpertoken(c["q"], c["kcache"], c["vcache"], c["block_ids"],
                                   c["kv_lens_total"], c["q_scale"], c["k_scale"], c["v_scale"],
                                   num_seq_q)


@pytest.mark.parametrize("num_batch", [1, 16, 200])
@pytest.mark.parametrize("num_seq_q", [1, 2, 3, 4])
@pytest.mark.parametrize("max_seq_kv", [1024, 4096])
@pytest.mark.parametrize("kv_head_q_head", [(1, 8), (4, 32)])
@pytest.mark.parametrize("layout", ["NHD", "HND"])
@pytest.mark.parametrize("use_dynamic_sched", [False, True])
def test_decode_fp8_kpertoken_vs_oracle(hpc, num_batch, num_seq_q, max_seq_kv, kv_head_q_head, layout,
                                        use_dynamic_sched):
    """Grid of reference tests/test_attention_decode_qkpertoken_perhead_vperhead_fp8.py:446-456
    (use_dynamic_sched=False = no caller task map), tolerance atol=0.1 (:443)."""
    hkv, hq = kv_head_q_head
    if num_batch == 200 and (max_seq_kv == 4096 or not use_dynamic_sched) and hkv == 4:
        pytest.skip("CPU oracle too slow for this cell; same kernel path as the smaller cells")
    g = torch.Generator().manual_seed(41)
    lens = torch.randint(1, max_seq_kv, (num_batch,), generator=g, dtype=torch.int32) + num_seq_q
    d = oa.make_decode_fp8_kpt_inputs(num_batch, num_seq_q, lens, hkv, hq, seed=41, layout=layout,
                                      device="cuda")
    my = _run_decode_kpt(hpc, d, num_batch, num_seq_q, hkv, use_task_map=use_dynamic_sched)
    _check(my, _oracle_kpt(d, num_seq_q), f"kpt B{num_batch} Sq{num_seq_q} S{max_seq_kv} {kv_head_q_head} {layout}",
           atol=0.1, rel_max=0.06)


@pytest.mark.parametrize("lens", [[1], [2, 64, 65, 127, 128, 129, 255, 256, 257], [40000], [131] * 37])
@pytest.mark.parametrize("num_seq_q", [1, 4])
def test_decode_fp8_kpertoken_edge_lengths(hpc, lens, num_seq_q):
    lens = [max(L, num_seq_q) for L in lens]
    B = len(lens)
    d = oa.make_decode_fp8_kpt_inputs(B, num_seq_q, lens, 2, 8, seed=7, device="cuda")
    for mpl in (64, 1024):
        my = _run_decode_kpt(hpc, d, B, num_seq_q, 2, min_process_len=mpl)
        _check(my, _oracle_kpt(d, num_seq_q), f"kpt lens {lens[:4]} Sq{num_seq_q} mpl{mpl}", atol=0.1, rel_max=0.06)


def test_decode_fp8_kpertoken_golden_fixtures(hpc):
    from test_oracle_attention import load_kpt

    for name in ("decode_fp8_kpt_b3_nhd.npz", "decode_fp8_kpt_b4_hnd.npz"):
        z, d, (B, sq, hkv, hq, D, bs), layout = load_kpt(name)
        kv = d["kvcache"].cuda()
        if layout == 1:
            kv = kv.permute(0, 1, 3, 2, 4).contiguous().permute(0, 1, 3, 2, 4)
        dd = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in d.items()}
        dd.update(kvcache=kv, kcache=kv[:, 0, :bs], vcache=kv[:, 1, :bs], k_scale=kv[:, 0, bs:])
        my = _run_decode_kpt(hpc, dd, B, sq, hkv)
        _check(my, torch.from_numpy(z["out"]), name, atol=0.1)


def test_decode_rejects_unsupported(hpc):
    d = oa.make_decode_fp8_inputs(2, 1, [100, 100], 2, 8, seed=1, device="cuda")
    with pytest.raises(RuntimeError):  # k scales that are not the cache's own rows
        hpc.attention_decode_fp8(d["q"], d["kvcache"][:, 0], d["kvcache"][:, 1], d["block_ids"],
                                 d["kv_lens_total"], d["q_scale"], d["k_scale"], d["v_scale"],
                                 quant_type=hpc.QuantType.QPERTOKEN_PERHEAD_KPERTOKEN_PERHEAD_VPERHEAD)
    with pytest.raises(RuntimeError):
        hpc.attention_decode_fp8(d["q"], d["kvcache"][:, 0], d["kvcache"][:, 1], d["block_ids"],
                                 d["kv_lens_total"], d["q_scale"], d["k_scale"], d["v_scale"],
                                 quant_type=hpc.QuantType.QPERTENSOR_KPERTENSOR_VPERTENSOR)
    with pytest.raises(RuntimeError):
        hpc.attention_decode_fp8(d["q"].float(), d["kvcache"][:, 0], d["kvcache"][:, 1],
                                 d["block_ids"], d["kv_lens_total"], d["q_scale"], d["k_scale"],
                                 d["v_scale"])
    from test_decode_bf16_gpu import _bad_outputs

    for bad, what in _bad_outputs(d["q"]):
        with pytest.raises(RuntimeError, match="output"):
            hpc.attention_decode_fp8(d["q"], d["kvcache"][:, 0], d["kvcache"][:, 1],
                                     d["block_ids"], d["kv_lens_total"], d["q_scale"],
                                     d["k_scale"], d["v_scale"], output=bad)
        torch.cuda.synchronize()
        assert bool((bad == 7).all()), f"{what}: written before the rejection"
