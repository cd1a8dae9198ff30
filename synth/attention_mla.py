"""Seeded inputs for the absorbed MLA decode (csrc/decode_attn_mla.cu, oracle/attention_mla.py).

A case is a dict: q [B*sq, H, 576] bf16, kv [blocks, 64, 576] bf16, block_ids [B, max_blocks]
int32 (pages in random order), lens_total [B] int32 (cached tokens, the sq new ones included),
num_seq_q, scale, chunks (the split-k chunks of every (request, query tile) pair of the decode
schedule, oracle.taskmap.pair_chunks with num_head_kv = T), min_process_len and num_total_ctas.

Every slot past a request's last token, and every page no request uses, holds NaN: a kernel that
lets one of them into the output fails on NaN, and in a V column it would enter through 0 * NaN.

Kinds (the scores are spread to |s| ~ 50 in all of them):
  wide  q and kv N(0, 1)-shaped: every key, page, MTP row and query tile carries weight
  pe    q_nope = 0: the scores are decided by the 64 k_pe columns alone (a kernel that drops the
        RoPE part of QK sees uniform scores)
  vhigh kv columns 0..447 are 0: the V pattern lives in columns 448..511 (a V column offset or a
        swapped / repeated O half moves it)
  needle one Hadamard direction per (request, query row) in the 512 latent columns; one visible
        key of the request holds it with score ln(len) + 6 over a background of std 1.5. With
        `seams` {(b, tile): keys} (oracle.decode_walk.seam_keys) the needles of a query tile's
        rows sit on those keys first, then on page and tile edges; `heads` {(b, tile): [(first,
        seam, end)]} with `climb` c adds c to the score of the head part [first, seam) of every
        split task through k_pe and a q_pe shared by all rows (c > 0: the head part's maximum
        above the tail's, c < 0 below).
"""
import math

import torch

from oracle import taskmap
from oracle.attention_mla import DQK, PAGE, num_tiles

KINDS = ("wide", "pe", "vhigh")  # "needle" is built for the walk tests (seams)
SCALE_DSV3 = (0.1 * math.log(40.0) + 1.0) ** 2 / math.sqrt(192.0)  # mscale^2 / sqrt(qk_head_dim)
SCALE_PLAIN = 1.0 / 16.0


def _needles(q, kv, block_ids, lens_total, h, sq, scale, g, seams, heads, climb):
    from synth.attention_exact import hadamard
    dirs = hadamard(512).float() / math.sqrt(512)  # unit rows
    c = 1.5 / (scale * math.sqrt(512))             # background score std 1.5
    u = torch.ones(64) / 8                          # the shared q_pe direction (unit)
    kv[..., 512:] *= 0.1
    q.zero_()
    rows = sq * h
    for b, n in enumerate(lens_total):
        a = (math.log(n) + 6.0) / (c * scale)
        keys = kv[block_ids[b, :(n + PAGE - 1) // PAGE].long()].reshape(-1, DQK)  # a copy
        for t in range((rows + 63) // 64):
            ranges = (heads or {}).get((b, t), []) if climb else []
            for lo, seam, _ in ranges:
                keys[lo:seam, 512:] += climb * u / scale
            front = list((seams or {}).get((b, t), [])) + [0, 63, 64, 127, 128, n // 2]
            used = set()
            for ri in range(64 * t, min(64 * t + 64, rows)):
                lim = n - sq + ri // h
                pos = next((k for k in front if k <= lim and k not in used), None)
                if pos is None:
                    pos = int(torch.randint(0, lim + 1, (1,), generator=g))
                used.add(pos)
                q[b * sq + ri // h, ri % h, :512] = c * dirs[ri]
                if ranges:
                    q[b * sq + ri // h, ri % h, 512:] = u
                keys[pos, :512] += a * dirs[ri]
        kv[block_ids[b, :(n + PAGE - 1) // PAGE].long()] = keys.reshape(-1, PAGE, DQK)


def make_case(lens_total, h, mtp, seed, kind="wide", scale=SCALE_DSV3, num_total_ctas=132,
              min_process_len=512, extra_blocks=3, seams=None, heads=None, climb=0.0):
    g = torch.Generator().manual_seed(seed)
    sq = mtp + 1
    nb = len(lens_total)
    lens = torch.tensor(lens_total, dtype=torch.int32)
    assert int(lens.min()) >= sq
    npg = [(int(n) + PAGE - 1) // PAGE for n in lens_total]
    max_blocks = max(npg)
    nblocks = sum(npg) + extra_blocks
    kv = torch.randn(nblocks, PAGE, DQK, generator=g)
    q = torch.randn(nb * sq, h, DQK, generator=g)
    spread = 15.0  # std of s; the extremes of a row reach ~50
    if kind == "pe":
        q[..., :512] = 0
        q *= spread / (math.sqrt(64) * scale)
    elif kind == "vhigh":
        kv[..., :448] = 0
        q *= spread / (math.sqrt(128) * scale)
    else:
        q *= spread / (math.sqrt(DQK) * scale)
    perm = torch.randperm(nblocks, generator=g).to(torch.int32)
    block_ids = torch.full((nb, max_blocks), -1, dtype=torch.int32)
    o = 0
    for b, n in enumerate(lens_total):
        block_ids[b, :npg[b]] = perm[o:o + npg[b]]
        o += npg[b]
    if kind == "needle":
        _needles(q, kv, block_ids, [int(n) for n in lens_total], h, sq, scale, g, seams, heads,
                 climb)
    kv = kv.to(torch.bfloat16)
    q = q.to(torch.bfloat16)
    used = torch.zeros(nblocks, dtype=torch.bool)
    for b, n in enumerate(lens_total):
        ids = block_ids[b, :npg[b]]
        used[ids.long()] = True
        tail = int(n) - (npg[b] - 1) * PAGE
        kv[int(ids[-1]), tail:] = math.nan
    kv[~used] = math.nan
    # unused block_ids entries point at a page of NaN (never read by a correct kernel)
    spare = int(perm[-1])
    block_ids[block_ids < 0] = spare
    T = num_tiles(h, sq)
    chunks = taskmap.pair_chunks(list(lens_total), num_total_ctas, T, sq, min_process_len)
    return dict(q=q, kv=kv, block_ids=block_ids, lens_total=lens, num_seq_q=sq, scale=scale,
                chunks=chunks, min_process_len=min_process_len, num_total_ctas=num_total_ctas,
                kind=kind, h=h, mtp=mtp)


def lengths(sq):
    """The length set of the main GPU cases: 1 key beyond the MTP rows, page and tile edges."""
    return [sq, sq + 1, 63, 64, 65, 127, 128, 129, 200, 777]
