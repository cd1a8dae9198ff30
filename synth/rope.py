"""Synthetic inputs for rope_norm_store_kv[_fp8] (distributions and padding of reference
tests/test_rope.py:15-32,122-225)."""
import torch


def generate_cos_sin_cache(max_position, head_dim, base=10000.0):
    inv_freq = 1.0 / (base ** (torch.arange(0, head_dim, 2).float() / head_dim))
    t = torch.arange(max_position).float()
    freqs = torch.outer(t, inv_freq)
    return torch.cat([freqs.cos(), freqs.sin()], dim=-1)


def make_inputs(num_req, is_prefill, mtp, num_q_heads, num_kv_heads, qk_head_dim, v_head_dim=None,
                kv_block_size=64, max_num_kv_blocks=256, max_rope_position=2048, seed=0,
                len_range=(20, 200), pad_decode=True):
    """Returns a dict of CPU tensors; decode batches are padded to a multiple of 8 requests / rows
    like a CUDA-graph batch (padding requests have length 0 and q_index == padded row count)."""
    g = torch.Generator().manual_seed(seed)
    v_head_dim = v_head_dim or qk_head_dim
    hidden = num_q_heads * qk_head_dim + num_kv_heads * (qk_head_dim + v_head_dim)
    cos_sin = generate_cos_sin_cache(max_rope_position, qk_head_dim)
    kcache = torch.randn(max_num_kv_blocks, kv_block_size, num_kv_heads, qk_head_dim, generator=g).to(torch.bfloat16)
    vcache = torch.randn(max_num_kv_blocks, kv_block_size, num_kv_heads, v_head_dim, generator=g).to(torch.bfloat16)
    qw = torch.randn(qk_head_dim, generator=g)
    kw = torch.randn(qk_head_dim, generator=g)
    lens = torch.randint(len_range[0], len_range[1], (num_req,), generator=g)
    if is_prefill:
        q_len = torch.minimum((torch.rand(num_req, generator=g) * lens).long() + 1, lens)
        total = lens
    else:
        q_len = torch.full((num_req,), mtp + 1)
        total = lens + mtp + 1
    rows = int(q_len.sum())
    qkv = torch.randn(rows, hidden, generator=g).to(torch.bfloat16)
    q_index = torch.zeros(num_req + 1, dtype=torch.int32)
    q_index[1:] = torch.cumsum(q_len, 0)
    nblk = (total + kv_block_size - 1) // kv_block_size
    perm = torch.randperm(max_num_kv_blocks, generator=g)
    kv_idx = torch.full((num_req, int(nblk.max()) + 4), -1, dtype=torch.int32)
    off = 0
    for i in range(num_req):
        kv_idx[i, :int(nblk[i])] = perm[off:off + int(nblk[i])]
        off += int(nblk[i])
    num_seqlen = total.to(torch.int32)
    real_rows = None
    if not is_prefill and pad_decode:
        real_rows = rows
        pb, pr = (num_req + 7) // 8 * 8, (rows + 7) // 8 * 8
        qkv = torch.cat([qkv, torch.zeros(pr - rows, hidden, dtype=qkv.dtype)])
        num_seqlen = torch.cat([num_seqlen, torch.zeros(pb - num_req, dtype=torch.int32)])
        q_index = torch.cat([q_index, torch.full((pb - num_req,), pr, dtype=torch.int32)])
        kv_idx = torch.cat([kv_idx, torch.zeros(pb - num_req, kv_idx.shape[1], dtype=torch.int32)])
    return dict(qkv=qkv, num_seqlen=num_seqlen, q_index=q_index, kcache=kcache, vcache=vcache,
                kv_indices=kv_idx, q_norm_w=qw, k_norm_w=kw, cos_sin=cos_sin, real_rows=real_rows,
                num_req=num_req)


# ---- inputs of the exact tests (tests/test_rope_exact_*.py) --------------------------------------
BF16_SENTINEL = 0x7FC0  # bf16 NaN: a cache slot nobody wrote still holds it
FP8_SENTINEL = 0x7F     # e4m3 NaN
GUARD_PAGE = 0          # page id of padding requests and of pages no row of the call writes


def random_cos_sin(max_position, head_dim, seed):
    """A cos | sin table drawn uniformly from [-1, 1] per (position, dim): reading a wrong
    position or dim changes every element."""
    g = torch.Generator().manual_seed(seed)
    return torch.rand(max_position, head_dim, generator=g) * 2 - 1


def _request_shape(c, g):
    """(q_len, ctx) per request and the number of padded requests / rows."""
    if c["mode"] == "prefill":
        q_len = [int(n) for n in c.get("q_lens", (7, 0, 40, 0, 1, 23))]
        ctx = [int(torch.randint(0, 3 * c["page"], (1,), generator=g)) for _ in q_len]
        ctx[3] = 0  # a request with no tokens at all
        return q_len, ctx, len(q_len), sum(q_len)
    sq = c["mtp"] + 1
    q_len = [sq] * c["batch"]
    ctx = [int(torch.randint(1, 4 * c["page"], (1,), generator=g)) for _ in q_len]
    if c.get("long"):
        ctx[-1] = 65536 + 3 * c["page"] + 5  # positions past 2^16
    rows = sum(q_len)
    return q_len, ctx, (c["batch"] + 7) // 8 * 8, (rows + 7) // 8 * 8


def make_exact_inputs(c):
    """CPU inputs of one exact-test case `c` (a dict, see tests/test_rope_exact_cpu.py):
    bf16 qkv whose heads alternate between unit scale and 2^-10 (there eps dominates the RMS),
    q and k norm weights with distinct halves, a random (or, with table="rotary", a real) cos/sin
    table, and the cache as ONE flat sentinel buffer that holds the K and V caches either as two
    separate [blocks, page, Hkv, D] tensors or interleaved as [blocks, 2, page, Hkv, D]
    (`cache_views`). Every request owns distinct pages except that pages no row writes in a long
    context map to GUARD_PAGE. Decode batches are padded to 8 requests / rows like a CUDA-graph
    batch (padding requests have length 0, q_index == padded row count, pages GUARD_PAGE)."""
    g = torch.Generator().manual_seed(c["seed"])
    hq, hkv, dqk, dv, page = c["hq"], c["hkv"], c["dqk"], c["dv"], c["page"]
    q_len, ctx, nreq, rows = _request_shape(c, g)
    lens = [a + b for a, b in zip(q_len, ctx)]
    hidden = hq * dqk + hkv * (dqk + dv)
    heads = hq + hkv
    x = torch.randn(rows, hidden, generator=g)
    scale = torch.ones(hidden)
    for h in range(1, heads, 3):
        scale[h * dqk:(h + 1) * dqk] = 2.0 ** -10
    qkv = (x * scale).to(torch.bfloat16)
    real = sum(q_len)
    qkv[real:] = 0
    max_pos = max(lens) + 2
    if c.get("table") == "rotary":
        cos_sin = generate_cos_sin_cache(max(max_pos, 4096), dqk)
    else:
        cos_sin = random_cos_sin(max(max_pos, 256), dqk, c["seed"] + 1)
    qw = 0.5 + torch.rand(dqk, generator=g)
    kw = 0.5 + torch.rand(dqk, generator=g)
    qw[dqk // 2:] += 1.0   # halves differ, and q differs from k
    kw[:dqk // 2] -= 0.25

    nblk = [(n + page - 1) // page for n in lens]
    max_blocks = max(nblk) + 2
    kv_idx = torch.full((nreq, max_blocks), GUARD_PAGE, dtype=torch.int32)
    nxt = 1
    for r, n in enumerate(nblk):
        first = (ctx[r] // page) if n > 64 else 0  # long context: only the written pages are real
        for b in range(first, n):
            kv_idx[r, b] = nxt
            nxt += 1
    num_pages = nxt + 2
    perm = torch.randperm(num_pages - 1, generator=g) + 1  # shuffle the real page ids, keep 0
    kv_idx = torch.where(kv_idx > 0, perm[(kv_idx - 1).clamp_min(0).long()].int(), kv_idx)

    q_index = torch.zeros(nreq + 1, dtype=torch.int32)
    q_index[1:len(q_len) + 1] = torch.cumsum(torch.tensor(q_len), 0).int()
    q_index[len(q_len) + 1:] = rows
    seqlen = torch.zeros(nreq, dtype=torch.int32)
    seqlen[:len(lens)] = torch.tensor(lens, dtype=torch.int32)

    k_page, v_page = page * hkv * dqk, page * hkv * dv
    if c["layout"] == "combined":
        assert dqk == dv
        geom = dict(k_off=0, v_off=k_page, k_stride=2 * k_page, v_stride=2 * k_page)
    else:
        geom = dict(k_off=0, v_off=num_pages * k_page, k_stride=k_page, v_stride=v_page)
    geom.update(num_pages=num_pages, flat=num_pages * (k_page + v_page), page=page, hq=hq, hkv=hkv,
                dqk=dqk, dv=dv, layout=c["layout"])
    return dict(qkv=qkv, cos_sin=cos_sin, num_seqlen=seqlen, q_index=q_index, kv_indices=kv_idx,
                q_norm_w=qw, k_norm_w=kw, geom=geom, is_prefill=c["mode"] == "prefill",
                max_seqlens=max(q_len), policy=c["policy"], real_rows=real)


def cache_views(flat, geom):
    """The K and V cache tensors the op receives, as views of the flat cache buffer: two
    separate caches, or `kvcache[:, 0]` / `kvcache[:, 1]` of one [blocks, 2, page, Hkv, D] cache
    (page stride 2 * page * Hkv * D)."""
    n, page, hkv, dqk, dv = geom["num_pages"], geom["page"], geom["hkv"], geom["dqk"], geom["dv"]
    if geom["layout"] == "combined":
        kv = flat.view(n, 2, page, hkv, dqk)
        return kv[:, 0], kv[:, 1]
    k = flat[:n * page * hkv * dqk].view(n, page, hkv, dqk)
    v = flat[n * page * hkv * dqk:].view(n, page, hkv, dv)
    return k, v


def at_offset(t, byte_offset):
    """A contiguous copy of `t` that starts `byte_offset` bytes into a fresh buffer (an
    `byte_offset` of 4 makes the pointer 4-byte but not 16-byte aligned)."""
    e = byte_offset // t.element_size()
    buf = torch.empty(t.numel() + e, dtype=t.dtype, device=t.device)
    out = buf[e:].view(t.shape)
    out.copy_(t)
    return out
