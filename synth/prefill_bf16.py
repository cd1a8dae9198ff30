"""Synthetic inputs of the bf16 prefill ops (attention_prefill_bf16, attention_with_kvcache_prefill_bf16).

* make_reference_case: the reference tests' distributions (q and k ~ N(0, 1) / sqrt(128), v ~ N(0, 1);
  randomly permuted pages). Their attention is near uniform, so outputs are near the mean of V and
  would pass with many wrong masks; they are used at the reference's tolerance only.
* make_exact_case: inputs whose O(1) outputs depend on Q, K, V and the masks:
  - "peaked": scores of standard deviation 2.5 (natural-log units), so each row weighs a few keys
    and the softmax scale, K and V all show in the output.
  - "needle": position codes. Key j of a request is (cos t_f j, sin t_f j) over 64 random
    frequencies t_f in (0, 0.8); query row i points at position c_i = b_i + 1/2, where
    b_i = skv - sq + i is its causal boundary, so its score is A mean_f cos(t_f (j - c_i)):
    the boundary key and the key one past it score highest (A cos(t_f / 2)), the rest fall off.
    The row's output is mostly V of its boundary key; seeing one key more or less, or keys of the
    wrong position, page, head or request, moves it by O(1).
  V is N(0, 1) per (token, kv head), so every kv head has its own V. Paged caches: pages are
  randomly permuted and the unused tail of each request's last page holds poison (K that would
  outscore every key of the request's last row by 2A, V = 1000); unused pages are random.
GRID is the GPU test's list of cases; applicable() says which oracle mutations
(oracle.prefill_bf16.MUTATIONS) a case can show.
"""
import math

import torch

D = 128
NEEDLE_A = 24.0
POISON_V = 1000.0

# op, q lengths, kv lengths (paged), Hq, Hkv, page, layout, extra max_seqlens_q, seed
GRID = [
    dict(op="dense", q_lens=[1, 300, 0, 517, 128], hq=8, hkv=2, extra=200, seed=1),
    dict(op="dense", q_lens=[700, 45], hq=8, hkv=8, extra=0, seed=2),
    dict(op="dense", q_lens=[257, 1000], hq=16, hkv=2, extra=1, seed=3),
    dict(op="paged", q_lens=[1, 200, 0, 300], kv_lens=[1, 777, 50, 300], hq=8, hkv=2, page=16,
         layout="NHD", extra=0, seed=4),
    dict(op="paged", q_lens=[129, 400], kv_lens=[1500, 400], hq=16, hkv=2, page=32, layout="HND",
         extra=100, seed=5),
    dict(op="paged", q_lens=[513, 63], kv_lens=[1100, 255], hq=4, hkv=4, page=64, layout="NHD",
         extra=0, seed=6),
    dict(op="paged", q_lens=[333], kv_lens=[333], hq=4, hkv=1, page=64, layout="HND", extra=300,
         seed=7),
]
KINDS = ("peaked", "needle")


def case_id(c):
    s = f"{c['op']}-hq{c['hq']}-hkv{c['hkv']}-q{'_'.join(map(str, c['q_lens']))}"
    if c["op"] == "paged":
        s += f"-kv{'_'.join(map(str, c['kv_lens']))}-bs{c['page']}-{c['layout']}"
    return s


def applicable(c, mutation):
    """Whether case `c` can show `mutation` at all."""
    q_lens = c["q_lens"]
    kv_lens = c.get("kv_lens", q_lens)
    g = c["hq"] // c["hkv"]
    if mutation == "kv_head_mod":
        return g > 1 and c["hkv"] > 1
    if mutation == "top_left":
        return any(0 < q < kv for q, kv in zip(q_lens, kv_lens))
    if mutation == "swap_pages":
        return c["op"] == "paged" and any(q > 0 and kv > c["page"] for q, kv in zip(q_lens, kv_lens))
    if mutation == "tail_visible":
        return c["op"] == "paged" and any(q > 0 and kv % c["page"] for q, kv in zip(q_lens, kv_lens))
    if mutation == "dense_prev_offset":
        return c["op"] == "dense" and sum(q > 0 for q in q_lens[1:]) > 0
    if mutation == "causal_off_by_one":
        return any(q > 1 for q in q_lens)
    return True


def _cu(q_lens):
    return torch.tensor([0] + list(q_lens), dtype=torch.int32).cumsum(0).to(torch.int32)


def _pages(kv_lens, page, gen, extra=3):
    nblk = [(n + page - 1) // page for n in kv_lens]
    num_blocks = sum(nblk) + extra
    perm = torch.randperm(num_blocks, generator=gen).to(torch.int32)
    ids = torch.full((len(kv_lens), max(max(nblk), 1) + 1), -1, dtype=torch.int32)  # unused: -1
    cu = 0
    for b, n in enumerate(nblk):
        ids[b, :n] = perm[cu:cu + n]
        cu += n
    return ids, num_blocks


def _cache(num_blocks, page, hkv, layout):
    """A [blocks, page, Hkv, D] view: NHD contiguous, or HND storage seen through strides."""
    if layout == "NHD":
        return torch.empty(num_blocks, page, hkv, D, dtype=torch.float32)
    return torch.empty(num_blocks, hkv, page, D, dtype=torch.float32).transpose(1, 2)


def _needle_keys(n, freqs):
    pos = torch.arange(n, dtype=torch.float64)[:, None] * freqs[None, :]
    return torch.stack([pos.cos(), pos.sin()], -1).reshape(n, D)


def _needle_queries(centers, freqs):
    ang = centers[:, None] * freqs[None, :]
    return NEEDLE_A * math.sqrt(D) / freqs.numel() * torch.stack([ang.cos(), ang.sin()], -1).reshape(-1, D)


def make_exact_case(c, kind, device="cpu"):
    """Inputs of GRID case `c` for input family `kind`. Returns a dict with "op", q, k, v (dense)
    or kcache, vcache, block_ids, seqlens_kv (paged), cu_seqlens_q, seqlens_q, max_q."""
    gen = torch.Generator().manual_seed(1000 * c["seed"] + KINDS.index(kind))
    q_lens = c["q_lens"]
    kv_lens = c.get("kv_lens", q_lens)
    hq, hkv = c["hq"], c["hkv"]
    total = sum(q_lens)
    freqs = torch.rand(D // 2, generator=gen, dtype=torch.float64) * 0.8
    q = torch.empty(total, hq, D, dtype=torch.float64)
    ks, vs = [], []
    for b, (nq, nkv) in enumerate(zip(q_lens, kv_lens)):
        if kind == "peaked":
            ks.append(torch.randn(nkv, hkv, D, generator=gen, dtype=torch.float64))
            qb = 2.5 * torch.randn(nq, hq, D, generator=gen, dtype=torch.float64)
        else:
            ks.append(_needle_keys(nkv, freqs)[:, None, :].expand(nkv, hkv, D))
            centers = nkv - nq + torch.arange(nq, dtype=torch.float64) + 0.5
            qb = _needle_queries(centers, freqs)[:, None, :].expand(nq, hq, D)
        vs.append(torch.randn(nkv, hkv, D, generator=gen, dtype=torch.float64))
        s0 = sum(q_lens[:b])
        q[s0:s0 + nq] = qb
    bf = lambda t: t.to(torch.bfloat16).to(device)  # noqa: E731
    d = dict(op=c["op"], q=bf(q), cu_seqlens_q=_cu(q_lens).to(device),
             seqlens_q=torch.tensor(q_lens, dtype=torch.int32, device=device),
             max_q=max(q_lens) + c["extra"])
    if c["op"] == "dense":
        d.update(k=bf(torch.cat(ks)), v=bf(torch.cat(vs)))
        return d
    page = c["page"]
    ids, num_blocks = _pages(kv_lens, page, gen)
    kc, vc = _cache(num_blocks, page, hkv, c["layout"]), _cache(num_blocks, page, hkv, c["layout"])
    kc.copy_(torch.randn(kc.shape, generator=gen))
    vc.copy_(torch.randn(vc.shape, generator=gen))
    for b, nkv in enumerate(kv_lens):
        nblk = (nkv + page - 1) // page
        kpad = torch.zeros(nblk * page, hkv, D, dtype=torch.float64)
        vpad = torch.full((nblk * page, hkv, D), POISON_V, dtype=torch.float64)
        kpad[:nkv], vpad[:nkv] = ks[b], vs[b]
        if nkv < nblk * page and q_lens[b] > 0:  # poison for the request's last row
            kpad[nkv:] = 3 * q[sum(q_lens[:b]) + q_lens[b] - 1, 0] / math.sqrt(D) * (
                1.0 if kind == "needle" else 1.0 / 2.5)
        for j in range(nblk):
            kc[int(ids[b, j])] = kpad[j * page:(j + 1) * page].float()
            vc[int(ids[b, j])] = vpad[j * page:(j + 1) * page].float()
    d.update(kcache=kc.to(torch.bfloat16).to(device), vcache=vc.to(torch.bfloat16).to(device),
             block_ids=ids.to(device), seqlens_kv=torch.tensor(kv_lens, dtype=torch.int32, device=device))
    return d


def make_reference_case(op, q_lens, kv_lens=None, hq=4, hkv=1, page=64, layout="NHD", seed=41,
                        device="cpu"):
    """The reference tests' input distributions (tests/test_attention_prefill_bf16.py,
    tests/test_attention_with_kvcache_prefill_bf16.py), on ragged lengths."""
    gen = torch.Generator().manual_seed(seed)
    total = sum(q_lens)
    bf = lambda t: t.to(torch.bfloat16).to(device)  # noqa: E731
    d = dict(op=op, q=bf(torch.randn(total, hq, D, generator=gen) / math.sqrt(D)),
             cu_seqlens_q=_cu(q_lens).to(device),
             seqlens_q=torch.tensor(q_lens, dtype=torch.int32, device=device), max_q=max(q_lens))
    if op == "dense":
        d.update(k=bf(torch.randn(total, hkv, D, generator=gen) / math.sqrt(D)),
                 v=bf(torch.randn(total, hkv, D, generator=gen)))
        return d
    ids, num_blocks = _pages(kv_lens, page, gen)
    kc, vc = _cache(num_blocks, page, hkv, layout), _cache(num_blocks, page, hkv, layout)
    kc.copy_(torch.randn(kc.shape, generator=gen) / math.sqrt(D))
    vc.copy_(torch.randn(vc.shape, generator=gen))
    d.update(kcache=kc.to(torch.bfloat16).to(device), vcache=vc.to(torch.bfloat16).to(device),
             block_ids=ids.to(device), seqlens_kv=torch.tensor(kv_lens, dtype=torch.int32, device=device))
    return d
