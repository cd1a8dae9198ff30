"""Seeded inputs for the Stem block-mask stages (hpc/stem.py).

`make_inputs` builds a varlen batch over a paged FP8 cache: ragged and chunked requests (kv - q not
a multiple of 128), q_len < 128 and q_len = 0, pages of 32 or 64 tokens in NHD or HND layout,
per-token qscale (padded past the longest request) and per-token kscale or per-tensor scales that
are not 1. Page tails past kv_len and unused pages hold NaN, which no stage may read.

With `planted=True` the scores have a known answer and the budget is a real top-k: requests are
late chunks of a 25600-token prompt (pass `num_prompt_tokens` = the prompt, 200 blocks, the large
regime), so a row sees up to 200 key blocks against a budget of about 25-50. Every query aligns with
one direction d. The keys of each key block are one fp8 level (0.25 .. 15, 12.5 % apart) times d,
and three planted blocks per (request, kv head), outside the sink and the window and visible to
every row, carry d at level 64. Scores are therefore ordered by level: blocks of one level tie
exactly, in the kernel and in fp64 alike, and distinct levels are far apart. Every V row has the same
norm (random signs, one magnitude) and kv_len is a multiple of 128, so vbias is the same for every
block and cannot reorder the levels. kscale is constant (per tensor, or per token)"""
import numpy as np
import torch

NAN_E4M3 = 0x7F

# planted batch: two late chunks of one 25600-token prompt (kv - q not a multiple of 128) and an
# empty request
PLANTED = dict(q_lens=[512, 300, 0], kv_lens=[25600, 12800, 1024], prompt=[25600, 25600, 1024])

# (q_lens, kv_lens, Hq, Hkv, page, layout, quant_type, alpha): the GPU grid of stage checks
CASES = [
    ([300, 77, 0, 128], [300, 1000, 500, 3100], 8, 2, 64, "nhd", 1, 1.0),
    ([513, 40], [7000, 2090], 8, 2, 32, "hnd", 0, 0.5),
    ([1024], [1024], 16, 2, 64, "hnd", 1, 0.5),
    ([200, 129], [12000, 20900], 4, 4, 64, "nhd", 0, 1.0),
    ([256, 1], [24000, 300], 8, 1, 32, "nhd", 1, 0.5),
]


def _e4m3(x):
    return x.clamp(-448, 448).to(torch.float8_e4m3fn)


def make_inputs(q_lens, kv_lens, Hq, Hkv, page=64, layout="nhd", quant_type=1, seed=0,
                planted=False, qscale_extra=37):
    g = torch.Generator().manual_seed(seed)
    B, D = len(q_lens), 128
    total = sum(q_lens)
    max_q = max(q_lens) if q_lens else 0
    npg = [(L + page - 1) // page for L in kv_lens]
    num_blocks = sum(npg) + 5
    perm = torch.randperm(num_blocks, generator=g)[:sum(npg)].to(torch.int32)
    block_ids = torch.zeros(B, max(npg) + 2, dtype=torch.int32)
    cur = 0
    for i in range(B):
        block_ids[i, :npg[i]] = perm[cur:cur + npg[i]]
        cur += npg[i]

    if planted:
        assert all(L % 128 == 0 for L in kv_lens), "planted inputs need whole 128-token blocks"
        d2 = torch.where(torch.rand(D, generator=g) < 0.5, -1.0, 1.0)
        q = d2.expand(total, Hq, D).clone()
        levels = torch.tensor([float(2.0 ** e * (1 + m / 8)) for e in range(-2, 4) for m in range(8)])
        k = torch.zeros(num_blocks, page, Hkv, D)
        plants = []
        for i in range(B):
            nkb = kv_lens[i] // 128
            off = -(-(kv_lens[i] - q_lens[i]) // 128)
            per_head = []
            for h in range(Hkv):
                lev = levels[torch.randint(0, levels.numel(), (nkb,), generator=g)]
                cand = list(range(4, max(4, off - 4)))  # outside the sink; every row sees them
                pl = sorted(cand[j] for j in torch.randperm(len(cand), generator=g)[:3].tolist())
                for kb in pl:
                    lev[kb] = 64.0
                per_head.append(pl)
                rows = torch.arange(kv_lens[i])
                pid = block_ids[i, rows // page].long()
                k[pid, rows % page, h] = lev[rows // 128][:, None] * d2[None, :]
            plants.append(per_head)
        v = 0.5 * torch.where(torch.rand(num_blocks, page, Hkv, D, generator=g) < 0.5, -1.0, 1.0)
        qscale = torch.rand(B, Hq, max_q + qscale_extra, generator=g) * 0.05 + 0.05
    else:
        q = torch.randn(total, Hq, D, generator=g) * 2
        k = torch.randn(num_blocks, page, Hkv, D, generator=g) * 2
        v = torch.randn(num_blocks, page, Hkv, D, generator=g)
        # V norms vary by block so that vbias is not flat
        v = v * (torch.rand(num_blocks, 1, Hkv, 1, generator=g) * 3 + 0.2)
        qscale = torch.rand(B, Hq, max_q + qscale_extra, generator=g) * 0.2 + 0.01
        plants = None
    kc = _e4m3(k)
    vc = _e4m3(v)
    # poison: page tails past kv_len and unused pages
    used = torch.zeros(num_blocks, page, dtype=torch.bool)
    for i in range(B):
        rows = torch.arange(kv_lens[i])
        used[block_ids[i, rows // page].long(), rows % page] = True
    kc.view(torch.uint8)[~used] = NAN_E4M3
    vc.view(torch.uint8)[~used] = NAN_E4M3
    if layout == "hnd":
        kc = kc.transpose(1, 2).contiguous().transpose(1, 2)
        vc = vc.transpose(1, 2).contiguous().transpose(1, 2)
    if quant_type == 1:
        kscale = torch.rand(1, generator=g) + 0.5
        vscale = torch.rand(1, generator=g) + 0.5
    else:
        kscale = torch.rand(num_blocks, page // 32, Hkv, 32, generator=g) + 0.5
        vscale = torch.rand(Hkv, generator=g) + 0.5
    if planted:
        kscale = torch.full_like(kscale, 0.75)
    cu = torch.zeros(B + 1, dtype=torch.int32)
    cu[1:] = torch.cumsum(torch.tensor(q_lens, dtype=torch.int32), 0)
    return dict(q=_e4m3(q), kcache=kc, vcache=vc, qscale=qscale, kscale=kscale, vscale=vscale,
                kv_indices=block_ids, cu_seqlens_q=cu,
                q_seq_lens=torch.tensor(q_lens, dtype=torch.int32),
                kv_seq_lens=torch.tensor(kv_lens, dtype=torch.int32),
                quant_type=quant_type, plants=plants)


def adversarial_logits(B, H, max_qb, max_kb, seed=0):
    """bf16 logits with ties at every level, -0 / +0, +-inf, NaN and whole rows of -inf."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-6, 7, (B, H, max_qb, max_kb), generator=g).float() * 0.5
    r = torch.rand(x.shape, generator=g)
    x = torch.where(r < 0.05, torch.tensor(float("-inf")), x)
    x = torch.where((r >= 0.05) & (r < 0.07), torch.tensor(float("nan")), x)
    x = torch.where((r >= 0.07) & (r < 0.09), torch.tensor(float("inf")), x)
    x = torch.where((r >= 0.09) & (r < 0.12), torch.tensor(-0.0), x)
    x[:, :, ::7] = float("-inf")  # rows with no finite value
    return x.to(torch.bfloat16)
