"""GPU parity tests for bf16 paged decode attention (`hpc.attention_decode_bf16`, SURVEY.md §8 f1).

Through the public API (hpc.* -> C-ABI -> sm_90a kernel), checked against the CPU oracle
(oracle/attention.py:decode_bf16, pinned bit-exactly to the reference's own test function) at the
reference's tolerance (atol=0.016, reference tests/test_attention_decode_bf16.py:203) plus a
relative-L2 bound of our own.
"""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import attention as oa

pytestmark = pytest.mark.gpu
G = Path(__file__).resolve().parent / "golden"


# ------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------
def _run(hpc, d, num_batch, num_seq_q, hkv, min_process_len=64, use_task_map=True, cpu_assign=False,
         new_kv_included=True, output=None):
    lens = d["kv_lens_total"]
    arg_lens = lens if new_kv_included else lens - num_seq_q
    task_map = None
    if use_task_map:
        task_map = hpc.get_attention_decode_task_workspace(num_batch, int(lens.max()), hkv, min_process_len)
        hpc.assign_attention_decode_task(arg_lens.cpu() if cpu_assign else arg_lens, task_map, hkv,
                                         num_seq_q, new_kv_included, min_process_len)
    return hpc.attention_decode_bf16(
        d["q"], d["kvcache"][:, 0], d["kvcache"][:, 1], d["block_ids"], arg_lens,
        mtp=num_seq_q - 1, new_kv_included=new_kv_included, splitk=True, task_map=task_map,
        output=output)


def _oracle(d, num_seq_q):
    dc = {k: v.cpu() for k, v in d.items()}
    return oa.decode_bf16(dc["q"], dc["kvcache"][:, 0], dc["kvcache"][:, 1], dc["block_ids"],
                          dc["kv_lens_total"], num_seq_q)


def _check(my, gt, tag="", atol=0.016, rel_max=0.01):
    my = my.float().cpu()
    gt = gt.float().cpu()
    err = (my - gt).abs()
    rel = err.norm() / gt.norm().clamp_min(1e-6)
    assert torch.isfinite(my).all(), f"{tag}: non-finite output"
    assert torch.allclose(my, gt, atol=atol), f"{tag}: max abs err {err.max():.4f}"
    assert rel < rel_max, f"{tag}: relative error {rel:.4f}"


@pytest.mark.parametrize("num_batch", [1, 16, 100])
@pytest.mark.parametrize("num_seq_q", [1, 2, 3])
@pytest.mark.parametrize("max_seq_kv", [1024, 4096])
@pytest.mark.parametrize("block_size", [16, 32, 64])
@pytest.mark.parametrize("kv_head_q_head", [(1, 8), (4, 32)])
@pytest.mark.parametrize("layout", ["NHD", "HND"])
def test_decode_bf16_vs_oracle(hpc, num_batch, num_seq_q, max_seq_kv, block_size, kv_head_q_head,
                               layout):
    """Grid of reference tests/test_attention_decode_bf16.py:206-216, widened to the page sizes the
    entry accepts (src/attention/entry.cc:443)."""
    hkv, hq = kv_head_q_head
    if num_batch == 100 and (max_seq_kv == 4096 or block_size != 64) and hkv == 4:
        pytest.skip("CPU oracle too slow for this cell; the 16-request cells cover the shape")
    g = torch.Generator().manual_seed(41)
    lens = torch.randint(1, max_seq_kv, (num_batch,), generator=g, dtype=torch.int32) + num_seq_q
    d = oa.make_decode_bf16_inputs(num_batch, num_seq_q, lens, hkv, hq, block_size=block_size,
                                   seed=41, layout=layout, device="cuda")
    my = _run(hpc, d, num_batch, num_seq_q, hkv)
    _check(my, _oracle(d, num_seq_q),
           f"B{num_batch} Sq{num_seq_q} S{max_seq_kv} bs{block_size} {kv_head_q_head} {layout}")


@pytest.mark.parametrize("lens", [[1], [2, 15, 16, 17, 64, 65, 127, 128, 129, 255, 256, 257],
                                  [5, 5, 5], [40000], [129] * 5, [131] * 37])
@pytest.mark.parametrize("num_seq_q", [1, 4])
@pytest.mark.parametrize("block_size", [16, 64])
def test_decode_bf16_edge_lengths(hpc, lens, num_seq_q, block_size):
    """Ragged / boundary lengths: single token, page and tile multiples, tails shorter than
    num_seq_q, one request split over every CTA."""
    lens = [max(L, num_seq_q) for L in lens]
    B = len(lens)
    d = oa.make_decode_bf16_inputs(B, num_seq_q, lens, 2, 8, block_size=block_size, seed=7,
                                   device="cuda")
    gt = _oracle(d, num_seq_q)
    for mpl in (64, 1024):
        my = _run(hpc, d, B, num_seq_q, 2, min_process_len=mpl)
        _check(my, gt, f"lens {lens[:4]} Sq{num_seq_q} bs{block_size} mpl{mpl}")


@pytest.mark.parametrize("group_sq", [(4, 5), (8, 4), (4, 1), (8, 1)])
def test_decode_bf16_mtp_rows(hpc, group_sq):
    """Row counts up to the tile limit: mtp 4 with 4 heads per group (20 rows), mtp 3 with 8 (32)."""
    group, sq = group_sq
    hkv = 2
    d = oa.make_decode_bf16_inputs(6, sq, [700, 64, 129, 2000, 33, 1500], hkv, hkv * group,
                                   block_size=32, seed=3, device="cuda")
    _check(_run(hpc, d, 6, sq, hkv), _oracle(d, sq), f"group {group} Sq {sq}")


def test_decode_bf16_golden_fixtures(hpc):
    """Outputs of the reference's own test reference function (tests/golden/make_golden.py)."""
    for name in ("decode_bf16_b3_bs16_nhd.npz", "decode_bf16_b4_bs64_hnd.npz"):
        z = np.load(G / name)
        B, sq, hkv, hq, D, bs = map(int, z["meta"])
        kv = torch.from_numpy(z["kvcache"]).view(torch.bfloat16).cuda()
        if int(z["layout"][0]) == 1:
            kv = kv.permute(0, 1, 3, 2, 4).contiguous().permute(0, 1, 3, 2, 4)
        d = dict(q=torch.from_numpy(z["q"]).view(torch.bfloat16).cuda(), kvcache=kv,
                 block_ids=torch.from_numpy(z["block_ids"]).cuda(),
                 kv_lens_total=torch.from_numpy(z["kv_lens_total"]).cuda())
        _check(_run(hpc, d, B, sq, hkv), torch.from_numpy(z["out"]), name)


def _strided_q(q, extra_heads):
    """q as the leading columns of a fused [rows, (Hq + extra) * 128] qkv buffer."""
    rows, hq, d = q.shape
    buf = torch.randn(rows, (hq + extra_heads) * d, device=q.device).to(q.dtype)
    buf[:, :hq * d] = q.reshape(rows, -1)
    v = buf[:, :hq * d].view(rows, hq, d)
    assert v.stride(0) > hq * d
    return v


def _strided_output(like, extra, sentinel=7.0):
    """An output view whose rows are `extra` elements wider than [Hq, 128]; the buffer is filled
    with `sentinel`."""
    rows, hq, d = like.shape
    buf = torch.full((rows, hq * d + extra), sentinel, dtype=torch.bfloat16, device=like.device)
    return buf, buf[:, :hq * d].view(rows, hq, d)


def test_decode_bf16_entry_variants_agree(hpc):
    """No task map (scheduled inside the call), device-assigned map, CPU-assigned map, lengths
    passed without the new tokens, caller-provided output, q as a row-strided view of a fused qkv
    buffer, output as a row-strided view (split-k combine and the direct write of unsplit pairs):
    one result, and nothing written outside the output view."""
    d = oa.make_decode_bf16_inputs(16, 2, [777] * 16, 4, 32, block_size=32, seed=5, device="cuda")
    a = _run(hpc, d, 16, 2, 4, use_task_map=False)
    b = _run(hpc, d, 16, 2, 4, min_process_len=512)
    c = _run(hpc, d, 16, 2, 4, min_process_len=512, cpu_assign=True)
    e = _run(hpc, d, 16, 2, 4, min_process_len=512, new_kv_included=False)
    out = torch.empty_like(d["q"])
    f = _run(hpc, d, 16, 2, 4, min_process_len=512, output=out)
    assert f.data_ptr() == out.data_ptr()
    g = _run(hpc, dict(d, q=_strided_q(d["q"], 16)), 16, 2, 4, min_process_len=512)
    for t in (b, c, e, f, g):
        assert torch.equal(a, t)
    _check(a, _oracle(d, 2), "variants")
    # min_process_len 4096: bins of 32 tiles, so some pairs are split and some are not
    base = _run(hpc, d, 16, 2, 4, min_process_len=4096)
    for mpl, want in ((512, a), (4096, base)):
        buf, view = _strided_output(d["q"], 128)
        y = _run(hpc, d, 16, 2, 4, min_process_len=mpl, output=view)
        assert y.data_ptr() == view.data_ptr() and torch.equal(y, want)
        assert bool((buf[:, 32 * 128:] == 7.0).all()), "written outside the output view"


def test_decode_bf16_paging_invariance(hpc):
    """Relocating pages (different block_ids, same logical KV) leaves the output bit-identical."""
    B, hkv, hq = 8, 4, 32
    d = oa.make_decode_bf16_inputs(B, 1, [3000 + 17 * i for i in range(B)], hkv, hq, block_size=16,
                                   seed=11, device="cuda")
    base = _run(hpc, d, B, 1, hkv)
    nblk = d["kvcache"].shape[0]
    perm = torch.randperm(nblk, device="cuda")
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(nblk, device="cuda")
    d2 = dict(d)
    d2["kvcache"] = d["kvcache"][perm]
    d2["block_ids"] = inv[d["block_ids"].long()].to(torch.int32)
    assert torch.equal(base, _run(hpc, d2, B, 1, hkv))


def test_decode_bf16_rejects_bad_arguments(hpc):
    d = oa.make_decode_bf16_inputs(2, 1, [100, 200], 1, 8, seed=1, device="cuda")
    k, v = d["kvcache"][:, 0], d["kvcache"][:, 1]
    with pytest.raises(RuntimeError, match="head dim 128"):
        hpc.attention_decode_bf16(d["q"][..., :64].contiguous(), k, v, d["block_ids"], d["kv_lens_total"])
    with pytest.raises(RuntimeError, match="mtp"):
        hpc.attention_decode_bf16(d["q"], k, v, d["block_ids"], d["kv_lens_total"], mtp=5)
    with pytest.raises(RuntimeError, match="blocksize"):
        hpc.attention_decode_bf16(d["q"], k[:, :8], v[:, :8], d["block_ids"], d["kv_lens_total"])
    for bad, what in _bad_outputs(d["q"]):
        with pytest.raises(RuntimeError, match="output"):
            hpc.attention_decode_bf16(d["q"], k, v, d["block_ids"], d["kv_lens_total"], output=bad)
        torch.cuda.synchronize()
        assert bool((bad == 7).all()), f"{what}: written before the rejection"


def _bad_outputs(q):
    """Outputs both decode wrappers must reject before any launch, each filled with 7."""
    rows, hq, d = q.shape
    full = lambda *s, **kw: torch.full(s, 7, device=kw.get("device", "cuda"),  # noqa: E731
                                       dtype=kw.get("dtype", torch.bfloat16))
    return [
        (full(rows, hq, d, dtype=torch.float32), "float32"),
        (full(rows - 1, hq, d), "one row short"),
        (full(rows, hq, d, device="cpu"), "on the CPU"),
        (full(rows, hq, 2 * d)[:, :, :d], "head stride 256"),
        (full(rows * hq * d).as_strided((rows, hq, d), (hq * d - d, d, 1)), "overlapping rows"),
        (full(rows, hq * d + 16)[:, 4:4 + hq * d].view(rows, hq, d), "base not 16-byte aligned"),
        (full(rows, hq * d + 4)[:, :hq * d].view(rows, hq, d), "row stride not 16-byte aligned"),
    ]
