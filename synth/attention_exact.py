"""Synthetic FP8 (and bf16 decode) attention inputs whose outputs depend visibly on Q, K, the
scales and the masks.

The plain builders (synth/decode.py, synth/prefill.py) draw scores with a standard deviation of
about 0.005, so the softmax is uniform and the output is the mean of V whatever Q and K are.
These builders design the scores first (in natural-log units, s = q.k / sqrt(D) after
dequantisation) and then quantise Q, K and V the way the kernels' callers do:

* "peaked": random scores of standard deviation `temperature`.
* "needle" (decode): every (request, q head, MTP row) has its own Hadamard direction, and one
  key of the request holds that direction with score ln(len) + 3, so the output is mostly the V
  row of that key. Needles sit at keys 0, 63/64/65, 127/128/129, the middle of the request (a
  middle split-k chunk for long requests), the last token of a partial page, and the last visible
  key of every MTP row. Poison keys (score 30) sit where the kernel must not look: each row's
  future MTP tokens, the K slots past the request's length in its last page (their V is zero,
  which the API allows: only V's unused slots must be zero), and every 8th key of a request
  carries poison for the next request's rows (pages belonging to other requests).
* "kscale" (decode, k per token): K is the same vector for every token; only the per-token k
  scale picks the needle, at t % 64 in {0, 31, 32, 63} of a page that depends on the kv head.
* "sched" (prefill): scores climb `climb` log2 per 128-key tile and `slope` per key inside a tile,
  which drives the lazy reference maximum; keys above the causal diagonal inside the diagonal
  tile are then far above every visible key (upper-triangle poison).
All decode rows of an MTP group get different q scales (factors 1, 1/2, 1/sqrt 2, 1/2 sqrt 2 of
the code range), so q-scale indexing by token is visible. Prefill tiles that the block mask
skips, and tiles past the first extra one when the mask is narrower than the KV, carry poison
for exactly the (q head, Q tile) that skips them.
"""
import math

import torch

D = 128
PAGE = 64
TILE = 128
POISON = 30.0
MTP_Q_RANGE = (1.0, 0.5, 0.7071, 0.3536)


def hadamard(n=D):
    h = torch.ones(1, 1, dtype=torch.float64)
    while h.shape[0] < n:
        h = torch.cat([torch.cat([h, h], 1), torch.cat([h, -h], 1)], 0)
    return h


def _e4m3(x):
    return x.to(torch.float32).to(torch.float8_e4m3fn)


def _quant_rows(x, code_max):
    """Per-row (last dim) scale so that the row's largest code is code_max."""
    s = (x.abs().amax(-1) / code_max).clamp_min(1e-12)
    return _e4m3(x / s[..., None]), s.float()


def _place_pages(lens, gen, extra=4, page=PAGE):
    nblk = [(n + page - 1) // page for n in lens]
    num_blocks = sum(nblk) + len(lens) + extra
    perm = torch.randperm(num_blocks, generator=gen)[:sum(nblk)].to(torch.int32)
    ids = torch.zeros(len(lens), max(nblk), dtype=torch.int32)
    cu = 0
    for i, nb in enumerate(nblk):
        ids[i, :nb] = perm[cu:cu + nb]
        cu += nb
    return ids, num_blocks


def _needle_positions(n, sq, rows, gen, page=PAGE, front=None, rotate=0):
    """One distinct visible key per row; rows ordered (q head in group, MTP row). Rows of the
    first q head take the last visible key of their MTP row; the others take the keys of `front`,
    then the page and tile edges rotated by `rotate`, then (without `front`) the middle of the
    request, then the last token of a partial page."""
    edges = [0, page - 1, page, page + 1, 127, 128, 129]
    k = rotate % len(edges)
    cand = (list(front) + edges[k:] + edges[:k]) if front is not None else edges + [n // 2 + 7]
    if n % page:
        cand.append(n - 1)
    used, out = set(), []
    for r in range(rows):
        gi, i = divmod(r, sq)
        lim = n - sq + i
        pos = None
        if gi == 0 and lim not in used:
            pos = lim  # last visible key of each MTP row
        for c in cand:
            if pos is None and c <= lim and c not in used:
                pos = c
        free = [j for j in range(lim + 1) if j not in used] if pos is None else []
        if pos is None:  # a short request: share a key once every visible one is taken
            pos = free[int(torch.randint(0, len(free), (1,), generator=gen))] if free else lim
        used.add(pos)
        out.append(pos)
    return out


def make_decode_exact_inputs(kind, lens, num_seq_q, num_head_kv, num_head_q, k_per_token=False,
                             temperature=4.0, layout="NHD", seed=0, device="cpu", seams=None,
                             heads=None, climb=0.0):
    """Decode inputs in the format of synth.decode.make_decode_fp8_inputs (kv per tensor) or
    make_decode_fp8_kpt_inputs (k per token). kind: "peaked", "needle" or "kscale" (k per
    token only). lens include the num_seq_q new tokens.

    Needle kind, for the rotated bin walk (oracle.decode_walk): `seams` {(b, h): keys} puts the
    needles of the rows of pair (b, h) on those keys first (decode_walk.seam_keys: both sides of
    every seam, segment ends, tasks between save and restore), and `heads` {(b, h): [(first,
    seam, end)]} with `climb` c adds c to the score of every key of the head part [first, seam)
    of each split task, for all rows of the group: c > 0 puts the head part's maximum above the
    tail's, c < 0 below it, so a restore that rescales m, l or O wrongly moves the output."""
    gen = torch.Generator().manual_seed(seed)
    lens = [int(n) for n in lens]
    B, sq, hkv, hq = len(lens), num_seq_q, num_head_kv, num_head_q
    g = hq // hkv
    rows = g * sq
    H = hadamard()
    ids, nblocks = _place_pages(lens, gen)
    qf = torch.zeros(B, sq, hq, D, dtype=torch.float64)
    kf = torch.zeros(nblocks, PAGE, hkv, D, dtype=torch.float64)
    ckt = torch.ones(nblocks, PAGE, hkv, dtype=torch.float64)  # per-token multiplier ("kscale")
    if kind == "peaked":
        qf.normal_(generator=gen).mul_(temperature)
        kf.normal_(generator=gen)
    elif kind == "needle":
        assert rows <= 32
        kf.normal_(generator=gen)
        for b, n in enumerate(lens):
            dirs = H[(b % 4) * 32:(b % 4) * 32 + rows]
            nxt = H[((b + 1) % 4) * 32:((b + 1) % 4) * 32 + rows].sum(0) if B > 1 else None
            shared = H[(b % 4) * 32 + 31]  # orthogonal to dirs (rows < 32) and to nxt
            page = ids[b].long()
            for h in range(hkv):
                kv = kf[page, :, h].reshape(-1, D)  # this request's keys, a copy
                ranges = (heads or {}).get((b, h), []) if climb else []
                for r in range(rows):
                    gi, i = divmod(r, sq)
                    qf[b, i, h * g + gi] = dirs[r] + (shared if ranges else 0)
                for lo, seam, _ in ranges:
                    kv[lo:seam] += climb * shared / math.sqrt(D)
                front = seams.get((b, h)) if seams is not None else None
                pos = _needle_positions(n, sq, rows, gen, front=front)
                for r in range(rows):
                    gi, i = divmod(r, sq)
                    kv[pos[r]] += (math.log(n) + 3.0) * dirs[r] / math.sqrt(D)
                    kv[n - sq + i + 1:n] += POISON * dirs[r] / math.sqrt(D)  # future MTP tokens
                if nxt is not None and n > 3:
                    other = torch.arange(3, n, 8)
                    other = other[~torch.isin(other, torch.tensor(pos))]
                    kv[other] += POISON * nxt / math.sqrt(D)
                kf[page, :, h] = kv.reshape(-1, PAGE, D)
    elif kind == "kscale":
        assert k_per_token and rows <= 32
        for b, n in enumerate(lens):
            page = ids[b].long()
            for h in range(hkv):
                # directions depend on the kv head too: a q head read against another kv head's
                # K sees no needle
                dirs = H[((b + h) % 4) * 32:((b + h) % 4) * 32 + rows]
                for r in range(rows):
                    gi, i = divmod(r, sq)
                    qf[b, i, h * g + gi] = dirs[r]
                kf[page, :, h] = dirs.sum(0) / math.sqrt(D)
                c = torch.rand(len(page) * PAGE, generator=gen, dtype=torch.float64) * 2
                # the needle: t % 64 in {0, 31, 32, 63}, page chosen by head and request
                nvis = n - sq + 1
                npg = (nvis + PAGE - 1) // PAGE
                off = (0, 31, 32, 63)[(h + b) % 4]
                p = (h + 2 * b) % npg
                key = p * PAGE + off
                if key >= nvis:
                    key = (p * PAGE + min(off, nvis - 1 - p * PAGE))
                c[key] = math.log(n) + 3.0
                ckt[page, :, h] = c.reshape(-1, PAGE)
    else:
        raise ValueError(kind)
    # K slots past each request's length (V there is zero): score POISON for every row
    for b, n in enumerate(lens):
        if n % PAGE == 0:
            continue
        last = int(ids[b, (n + PAGE - 1) // PAGE - 1])
        for h in range(hkv):
            if kind == "kscale":
                ckt[last, n % PAGE:, h] = POISON
            else:
                qr = qf[b, :, h * g:(h + 1) * g].reshape(-1, D)
                qr = qr / (qr * qr).sum(-1, keepdim=True)
                kf[last, n % PAGE:, h] += POISON * math.sqrt(D) * qr.sum(0)

    # ---- quantise: q per (token, head) with a different code range per MTP row ----
    qrange = torch.tensor([400.0 * MTP_Q_RANGE[i % 4] for i in range(sq)], dtype=torch.float64)
    q8, qs = _quant_rows(qf, qrange[None, :, None])
    v = torch.randn(nblocks, PAGE, hkv, D, generator=gen, dtype=torch.float64) * 2
    for b, n in enumerate(lens):
        if n % PAGE:
            last = int(ids[b, (n + PAGE - 1) // PAGE - 1])
            v[last, n % PAGE:] = 0  # API contract: unused V slots are zero
    v8 = _e4m3(v)
    if k_per_token:
        srows = PAGE * 4 // D
        amax = kf.abs().amax(-1).clamp_min(1e-12)  # [blocks, bs, hkv]
        k8 = _e4m3(kf / amax[..., None] * 448)
        kscale = (amax / 448 * ckt).float()  # [blocks, bs, hkv]
        rows_ = (kscale.permute(0, 2, 1).contiguous().view(torch.float8_e4m3fn)
                 .reshape(nblocks, hkv, srows, D).permute(0, 2, 1, 3))
        kvcache = torch.zeros(nblocks, 2, PAGE + srows, hkv, D, dtype=torch.float8_e4m3fn)
        kvcache[:, 0, :PAGE] = k8
        kvcache[:, 0, PAGE:] = rows_
        kvcache[:, 1, :PAGE] = v8
        v_scale = (torch.rand(hkv, generator=gen) * 0.5 + 0.05).float()
    else:
        ks = float(kf.abs().max()) / 448
        kvcache = torch.stack([_e4m3(kf / ks), v8], 1)
        k_scale = torch.tensor([ks], dtype=torch.float32)
        v_scale = (torch.rand(1, generator=gen) * 0.5 + 0.05).float()
    if layout == "HND":
        kvcache = kvcache.permute(0, 1, 3, 2, 4).contiguous().permute(0, 1, 3, 2, 4)
    dev = torch.device(device)
    kvcache = kvcache.to(dev)
    out = dict(q=q8.reshape(B * sq, hq, D).to(dev), q_scale=qs.reshape(B * sq, hq).to(dev),
               kvcache=kvcache, v_scale=v_scale.to(dev), block_ids=ids.to(dev),
               kv_lens_total=torch.tensor(lens, dtype=torch.int32, device=dev))
    if k_per_token:
        out.update(kcache=kvcache[:, 0, :PAGE], vcache=kvcache[:, 1, :PAGE],
                   k_scale=kvcache[:, 0, PAGE:])
    else:
        out.update(k_scale=k_scale.to(dev))
    return out


def _chunk_needles(chunks, page):
    """Keys a needle should sit on for a pair split into `chunks` [(start, keys)]: the first key
    of page 32 of the first chunk longer than 32 pages (the decode producer fetches page ids 32 at
    a time) and a key inside a middle chunk."""
    out = []
    for st, n in chunks:
        if n > 32 * page:
            out.append(st + 32 * page)
            break
    if len(chunks) > 1:
        st, n = chunks[len(chunks) // 2] if len(chunks) > 2 else chunks[1]
        out.append(st + n // 2 + 1)
    return out


def make_decode_bf16_exact_inputs(kind, lens, num_seq_q, num_head_kv, num_head_q, page,
                                  temperature=4.0, layout="NHD", chunks=None, seed=0,
                                  device="cpu"):
    """BF16 paged decode inputs in the format of synth.decode.make_decode_bf16_inputs, pages of
    `page` tokens; lens include the num_seq_q new tokens. kind "peaked" (random scores of standard
    deviation `temperature`) or "needle" (one Hadamard direction per (request, q head, MTP row),
    and one key of the request holds it with score ln(len) + 3). Needles sit at the keys of
    _needle_positions for this page size, at the last visible key of every MTP row and, given
    `chunks` (oracle.taskmap.pair_chunks of the schedule the call will use), inside a middle
    split-k chunk and on the first key of page 32 of a chunk longer than 32 pages. Poison (score
    30) sits on each row's future MTP tokens, on every 8th key of a request for the next
    request's rows, and, in both kinds, on the K slots past each request's length in its last
    page. Their V slots are zero, as the API requires; poison goes in K only. The returned
    "needles" maps (request, kv head) to the needle key of each row (rows ordered (q head in
    group, MTP row))."""
    gen = torch.Generator().manual_seed(seed)
    lens = [int(n) for n in lens]
    B, sq, hkv, hq = len(lens), num_seq_q, num_head_kv, num_head_q
    g = hq // hkv
    rows = g * sq
    H = hadamard()
    ids, nblocks = _place_pages(lens, gen, page=page)
    qf = torch.zeros(B, sq, hq, D, dtype=torch.float64)
    kf = torch.zeros(nblocks, page, hkv, D, dtype=torch.float64)
    needles = {}
    if kind == "peaked":
        qf.normal_(generator=gen).mul_(temperature)
        kf.normal_(generator=gen)
    elif kind == "needle":
        assert rows <= 32
        kf.normal_(generator=gen)
        for b, n in enumerate(lens):
            dirs = H[(b % 4) * 32:(b % 4) * 32 + rows]
            nxt = H[((b + 1) % 4) * 32:((b + 1) % 4) * 32 + rows].sum(0) if B > 1 else None
            pg = ids[b, :(n + page - 1) // page].long()
            for h in range(hkv):
                kv = kf[pg, :, h].reshape(-1, D)  # this request's keys, a copy
                for r in range(rows):
                    gi, i = divmod(r, sq)
                    qf[b, i, h * g + gi] = dirs[r]
                front = _chunk_needles(chunks[(b, h)], page) if chunks is not None else None
                pos = _needle_positions(n, sq, rows, gen, page, front, (b * hkv + h) * (rows - sq))
                needles[(b, h)] = pos
                for r in range(rows):
                    gi, i = divmod(r, sq)
                    kv[pos[r]] += (math.log(n) + 3.0) * dirs[r] / math.sqrt(D)
                if nxt is not None and n > 3:
                    other = torch.arange(3, n, 8)
                    other = other[~torch.isin(other, torch.tensor(pos))]
                    kv[other] += POISON * nxt / math.sqrt(D)
                kf[pg, :, h] = kv.reshape(-1, page, D)
    else:
        raise ValueError(kind)
    # future MTP tokens: key n - sq + j scores POISON for the rows i < j of its head group and
    # nothing extra for the others (K through the pseudo-inverse of the group's query rows)
    for b, n in enumerate(lens):
        for h in range(hkv):
            qg = qf[b, :, h * g:(h + 1) * g].transpose(0, 1).reshape(-1, D)  # rows (q head, MTP row)
            mtp_row = torch.arange(rows) % sq
            for j in range(1, min(sq, n)):
                t = n - sq + j
                want = POISON * math.sqrt(D) * (mtp_row < j).double()
                kf[ids[b, t // page], t % page, h] += (torch.linalg.pinv(qg) @ want)
    v = torch.randn(nblocks, page, hkv, D, generator=gen, dtype=torch.float64)
    for b, n in enumerate(lens):
        if n % page == 0:
            continue
        last = int(ids[b, (n + page - 1) // page - 1])
        v[last, n % page:] = 0  # API contract: unused V slots are zero
        for h in range(hkv):  # K slots past the length: score POISON for every row
            qr = qf[b, :, h * g:(h + 1) * g].reshape(-1, D)
            qr = qr / (qr * qr).sum(-1, keepdim=True)
            kf[last, n % page:, h] += POISON * math.sqrt(D) * qr.sum(0)
    kvcache = torch.stack([kf, v], 1).to(torch.bfloat16)
    if layout == "HND":
        kvcache = kvcache.permute(0, 1, 3, 2, 4).contiguous().permute(0, 1, 3, 2, 4)
    dev = torch.device(device)
    return dict(q=qf.reshape(B * sq, hq, D).to(torch.bfloat16).to(dev), kvcache=kvcache.to(dev),
                block_ids=ids.to(dev), kv_lens_total=torch.tensor(lens, dtype=torch.int32, device=dev),
                needles=needles)


def make_prefill_exact_inputs(q_lens, kv_lens, num_head_q, num_head_kv, skip, k_per_token,
                              kind="peaked", temperature=4.0, climb=0.7, slope=0.25, layout="nhd",
                              seed=0, mask_cols=None, dead_tile=None):
    """Prefill inputs in the format of synth.prefill.make_inputs. kind "peaked" (random scores of
    std `temperature`) or "sched" (scores climb `climb` log2 per KV tile and `slope` nat per key
    inside a tile, plus noise of std 0.5). skip: block-mask skip ratio or None (no mask);
    mask_cols: mask narrower than the KV; dead_tile (b, q head, Q tile): a Q tile whose every KV
    tile is masked (its rows are NaN, as in the reference)."""
    from synth.prefill import generate_block_sparse_mask

    gen = torch.Generator().manual_seed(seed)
    B, hq, hkv = len(q_lens), num_head_q, num_head_kv
    g = hq // hkv
    H = hadamard()
    bg = H[65:]  # 63 background directions; 0 = tile level, 1..64 = skip poison
    total, max_q = sum(q_lens), max(q_lens)
    nrow = (max_q + TILE - 1) // TILE
    ids, nblocks = _place_pages(kv_lens, gen, extra=2)

    t_bg = temperature if kind == "peaked" else 0.5
    a = t_bg / math.sqrt(D / bg.shape[0])
    qf = (torch.randn(total, hq, bg.shape[0], generator=gen, dtype=torch.float64) @ bg) * (
        a / math.sqrt(bg.shape[0]))
    kf = (torch.randn(nblocks, PAGE, hkv, bg.shape[0], generator=gen, dtype=torch.float64) @ bg) / (
        math.sqrt(bg.shape[0]))
    mask = None
    if skip is not None:
        ncol = mask_cols if mask_cols is not None else (max(kv_lens) + TILE - 1) // TILE
        mask = generate_block_sparse_mask(B, hq, nrow, ncol, skip, True, gen)
        if dead_tile is not None:
            mask[dead_tile] = False
        assert hq * nrow <= 64
    cu = [0]
    for n in q_lens:
        cu.append(cu[-1] + n)
    for b in range(B):
        nq, nkv = q_lens[b], kv_lens[b]
        page = ids[b].long()
        for h in range(hkv):
            kv = kf[page, :, h].reshape(-1, D)
            j = torch.arange(kv.shape[0], dtype=torch.float64)
            if kind == "sched":
                f = climb * math.log(2) * torch.div(j, TILE, rounding_mode="floor") + slope * (j % TILE)
                kv += f[:, None] * H[0] / math.sqrt(D)
                fmax = float(f[:nkv].max())
            else:
                fmax = 0.0
            if mask is not None:
                for hh in range(h * g, (h + 1) * g):
                    for m in range((nq + TILE - 1) // TILE):
                        last = (nkv - nq + min(nq, (m + 1) * TILE) - 1) // TILE
                        for n_ in range(last + 1):
                            seen = bool(mask[b, hh, m, n_]) if n_ < mask.shape[-1] else n_ == mask.shape[-1]
                            if not seen:
                                kv[n_ * TILE:(n_ + 1) * TILE] += ((fmax + POISON) / math.sqrt(D)
                                                                   * H[1 + hh * nrow + m])
            kf[page, :, h] = kv.reshape(-1, PAGE, D)
        for hh in range(hq):
            if kind == "sched":
                qf[cu[b]:cu[b + 1], hh] += H[0]
            if mask is not None:
                for m in range((nq + TILE - 1) // TILE):
                    qf[cu[b] + m * TILE:cu[b] + min(nq, (m + 1) * TILE), hh] += H[1 + hh * nrow + m]

    u = torch.rand(total, hq, generator=gen, dtype=torch.float64) * 0.6 + 0.4
    q8, qs_rows = _quant_rows(qf, 400.0 * u)
    pad = (max_q + TILE - 1) // TILE * TILE
    qscale = torch.ones(B, hq, pad, dtype=torch.float32)
    for b in range(B):
        qscale[b, :, :q_lens[b]] = qs_rows[cu[b]:cu[b + 1]].transpose(0, 1)
    v8 = _e4m3(torch.randn(nblocks, PAGE, hkv, D, generator=gen, dtype=torch.float64) * 2)
    if k_per_token:
        amax = kf.abs().amax(-1).clamp_min(1e-12)  # [blocks, bs, hkv]
        k8 = _e4m3(kf / amax[..., None] * 448)
        kscale = (amax / 448).float().reshape(nblocks, PAGE // 32, 32, hkv).permute(0, 1, 3, 2)
        kscale = kscale.contiguous()
        vscale = (torch.rand(hkv, generator=gen) * 0.5 + 0.05).float()
    else:
        ks = float(kf.abs().max()) / 448
        k8 = _e4m3(kf / ks)
        kscale = torch.tensor([ks], dtype=torch.float32)
        vscale = (torch.rand(1, generator=gen) * 0.5 + 0.05).float()
    if layout == "hnd":
        k8 = k8.transpose(1, 2).contiguous().transpose(1, 2)
        v8 = v8.transpose(1, 2).contiguous().transpose(1, 2)
    return dict(q=q8, kcache=k8, vcache=v8, qscale=qscale, kscale=kscale, vscale=vscale,
                cu_seqlens_q=torch.tensor(cu, dtype=torch.int32),
                seqlens_kv=torch.tensor(kv_lens, dtype=torch.int32), block_ids=ids,
                block_mask=mask, max_q=max_q)
