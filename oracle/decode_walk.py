"""ORACLE — test infrastructure only (see oracle/__init__.py).

CPU restatement of the rotated bin walk of the FP8 and MLA decode kernels (csrc/decode_common.cuh:
walk_start, scan_bin, segment_of), line for line, over a packed task map of oracle.taskmap.assign
whose header int 6 holds TB (tiles per kv head), as the device scheduler writes it and as
hpc/attention.py splices it into a CPU map.

walk(tm) gives, per CTA, the ordered segments it runs: the task row, its (request, kv head or
query tile) pair, chunk, tile range [tb, te), save / restore and how the task is written ("direct"
bf16 for a single-chunk pair, "split" for a partial of a split pair, None for the saved first part).
labels() names the walk paths a CTA takes:

  a   not rotated (u0 == 0)
  b   rotated at a task boundary (o == 0, ks > 0)
  c   single-row split: the bin's only task runs as [o, n) then [0, o)
  d   multi-row split; d:first / d:last / d:only give the split task's chunk role (chunk 0 of
      a split pair, its last chunk, the only chunk of its pair: a direct bf16 write). A middle
      chunk fills its whole bin, so a walk split inside one is single-row (c): d:middle cannot
      occur.
  e   the seam is one tile from either end of the split task (o == 1 or o == n - 1)
  f   a bin of more than 32 rows whose start row is 32 or beyond (second ballot round)
  g   short-bin fallback: u0 lies past the bin's last tile, the walk runs front to back
  h   the split task is causal for MTP rows (sq > 1); h:spill when the causal window of the pair's
      last chunk spills into the split task (the scheduler's F_IS_CAUSAL back-patching)

MUTATIONS restate walk bugs as per-key weights of one pair (mutant()), evaluated in fp64 on the
pair's own scores and values and written over the lossy oracle's output.
"""
import math
import random

import numpy as np
import torch

from oracle import taskmap

ROW = 12
TILE = 128
PATHS = ("a", "b", "c", "d", "e", "f", "g", "h")
SUBPATHS = ("d:first", "d:last", "d:only", "h:spill")
MUTATIONS = ("seam_tile_dropped", "seam_tile_twice", "carry_lost", "l_not_carried",
             "restore_wrong_target", "fallback_not_taken")


def header_tiles(lens, num_seq_q, new_kv_included=True, tilen=TILE):
    """Header int 6 as hpc/attention.py computes it for a CPU map (tiles per kv head)."""
    ns = np.asarray(lens, dtype=np.int64) + (0 if new_kv_included else num_seq_q)
    return int(((ns + tilen - 1) // tilen).sum())


def task_map(lens, num_ctas, num_head_kv, num_seq_q, min_process_len, new_kv_included=True):
    """oracle.taskmap.assign with header int 6 set."""
    tm = taskmap.assign(lens, num_ctas, num_head_kv, num_seq_q, TILE, new_kv_included,
                        min_process_len)
    tm[0, 6] = header_tiles(lens, num_seq_q, new_kv_included)
    return tm


def walk_start(tm, icta):
    P = int(tm[0, 0]) - 1
    TB = int(tm[0, 6])
    if TB <= 0 or P <= 0:
        return 0
    c = ((icta * P) % TB) % P
    return (P - c) % P


def scan_bin(bin_rows, max_rows, u0):
    """(m, ks, o, found) of scan_bin: 32-row ballot rounds, the first hit, the fallback."""
    if u0 <= 0:
        return max_rows, 0, 0, False
    m, before, found, ks, o = 0, 0, False, 0, 0
    for base in range(0, max_rows, 32):
        valid, c = [], []
        for lane in range(32):
            i = base + lane
            ok = i < max_rows and bin_rows[i, 0] >= 0 and bin_rows[i, 1] >= 0
            valid.append(ok)
            c.append(int(bin_rows[i, 6]) if ok else 0)
        cnt = 32 if all(valid) else valid.index(False)
        c = [c[l] if l < cnt else 0 for l in range(32)]
        excl = [before + sum(c[:l]) for l in range(32)]
        hits = [l for l in range(32) if l < cnt and excl[l] <= u0 < excl[l] + c[l]]
        if hits and not found:
            ks, o, found = base + hits[0], u0 - excl[hits[0]], True
        before += sum(c)
        m += cnt
        if cnt < 32:
            break
    if not found:
        ks, o = 0, 0
    return m, ks, o, found


def segment_of(m, ks, o, j):
    r = ks + j
    if r >= m:
        r -= m
    return dict(row=r, tb=o if j == 0 else 0, te=o if j == m else -1, save=o > 0 and j == 0,
                restore=j == m)


def _chunk_table(tm, num_batch, num_head_kv):
    ntpc1, ctas = int(tm[0, 0]), int(tm[0, 1])
    return tm[1 + ntpc1 * ctas:].reshape(-1)[:num_batch * num_head_kv]


def walk(tm, num_batch, num_head_kv, rotate=True, mutation=None):
    """Per CTA: dict(u0, m, ks, o, found, segs). Each segment: the walk fields plus h, b, chunk,
    start (first key of the task), keys, tiles, causal, kvcache (F_NUM_SEQKVCACHE), nchunks and
    write ("direct", "split" or None). `mutation` "fallback_not_taken": a CTA whose u0 is not
    found in its bin runs nothing."""
    ntpc1, ctas = int(tm[0, 0]), int(tm[0, 1])
    chunks = _chunk_table(tm, num_batch, num_head_kv)
    out = []
    for icta in range(ctas):
        rows = tm[1 + icta * ntpc1:1 + (icta + 1) * ntpc1]
        u0 = walk_start(tm, icta) if rotate else 0
        m, ks, o, found = scan_bin(rows, ntpc1 - 1, u0)
        nseg = m + (1 if o > 0 else 0)
        segs = []
        if not (mutation == "fallback_not_taken" and u0 > 0 and not found):
            for j in range(nseg):
                s = segment_of(m, ks, o, j)
                r = rows[s["row"]]
                if r[0] < 0 or r[1] < 0:  # the kernels' load_task: a terminator ends the walk
                    break
                h, b = int(r[0]), int(r[1])
                nch = int(chunks[h * num_batch + b])
                s.update(h=h, b=b, chunk=int(r[2]), start=int(r[3]), keys=int(r[4]),
                         kvcache=int(r[5]), tiles=int(r[6]), causal=int(r[8]), nchunks=nch,
                         write=None if s["save"] else ("direct" if nch == 1 else "split"))
                segs.append(s)
        out.append(dict(u0=u0, m=m, ks=ks, o=o, found=found, segs=segs))
    return out


def split_task(w):
    """The segment that saves (first part of the split task) of a CTA walk, or None."""
    return w["segs"][0] if w["segs"] and w["segs"][0]["save"] else None


def labels(w, num_seq_q):
    """The paths (PATHS, SUBPATHS) one CTA walk takes."""
    out = set()
    if w["u0"] == 0:
        out.add("a")
        return out
    if not w["found"]:
        if w["m"] > 0:
            out.add("g")
        return out
    if w["o"] == 0:
        out.add("b")
    if w["m"] > 32 and w["ks"] >= 32:
        out.add("f")
    s = split_task(w)
    if s is None:
        return out
    out.add("c" if w["m"] == 1 else "d")
    if w["m"] > 1:
        if s["nchunks"] == 1:
            out.add("d:only")
        elif s["chunk"] == 0:
            out.add("d:first")
        elif s["chunk"] == s["nchunks"] - 1:
            out.add("d:last")
        else:
            out.add("d:middle")
    if w["o"] in (1, s["tiles"] - 1):
        out.add("e")
    if s["causal"] and num_seq_q > 1:
        out.add("h")
        if s["chunk"] < s["nchunks"] - 1:
            out.add("h:spill")
    return out


def path_counts(walks, num_seq_q):
    """{path: number of CTAs that take it}."""
    cnt = {}
    for w in walks:
        for p in labels(w, num_seq_q):
            cnt[p] = cnt.get(p, 0) + 1
    return cnt


def pair_chunks(walks):
    """{(b, h): [(start, keys), ...]} in chunk order, from the walk's segments (each task once)."""
    out = {}
    for w in walks:
        for s in w["segs"]:
            if not s["save"]:
                out.setdefault((s["b"], s["h"]), []).append((s["chunk"], s["start"], s["keys"]))
    return {k: [(st, n) for _, st, n in sorted(v)] for k, v in out.items()}


def visits(walks):
    """{(b, h, chunk): [tile, ...]} in the order the walk runs them."""
    out = {}
    for w in walks:
        for s in w["segs"]:
            te = s["tiles"] if s["te"] < 0 else s["te"]
            out.setdefault((s["b"], s["h"], s["chunk"]), []).extend(range(s["tb"], te))
    return out


def seam_keys(walks):
    """Keys a needle should sit on, per (b, h), most telling first: the last key of tile o - 1
    and the first key of tile o of every split task; then the first and last key of the first
    and last tile of every segment, and a key in the middle of every task that runs between a
    save and its restore."""
    first_rank, rest = {}, {}

    def add(d, b, h, k, end):
        if 0 <= k < end:
            d.setdefault((b, h), []).append(k)

    for w in walks:
        segs = w["segs"]
        split = split_task(w) is not None
        for j, s in enumerate(segs):
            end = s["start"] + s["keys"]
            te = s["tiles"] if s["te"] < 0 else s["te"]
            first, last = s["start"] + s["tb"] * TILE, min(s["start"] + te * TILE, end) - 1
            if s["save"]:
                add(first_rank, s["b"], s["h"], first - 1, end)
                add(first_rank, s["b"], s["h"], first, end)
            for k in (first, min(first + TILE, end) - 1, max(last - TILE + 1, first), last):
                add(rest, s["b"], s["h"], k, end)
            if split and 0 < j < len(segs) - 1:
                add(rest, s["b"], s["h"], s["start"] + s["keys"] // 2, end)
    out = {}
    for k in set(first_rank) | set(rest):
        out[k] = list(dict.fromkeys(first_rank.get(k, []) + rest.get(k, [])))
    return out


def head_ranges(walks):
    """{(b, h): [(first key of the task, seam key, end of the task)]} of every split task: its
    head part [first, seam) runs last, its tail [seam, end) first."""
    out = {}
    for w in walks:
        s = split_task(w)
        if s is not None:
            out.setdefault((s["b"], s["h"]), []).append(
                (s["start"], s["start"] + w["o"] * TILE, s["start"] + s["keys"]))
    return out


# ------------------------------------------------------------------------------------------------
# path catalogue
# ------------------------------------------------------------------------------------------------
# FP8: (hkv, sq, group), rows = group * sq <= 16 (the kernel rotates for rows <= 16, an even
# hkv >= 2 and a token-major cache); MLA: (T, sq) for h128 mtp0, h64 mtp3, h128 mtp3
FP8_CONFIGS = [(2, 1, 4), (4, 2, 4), (8, 1, 8), (2, 3, 4), (4, 4, 4), (8, 2, 8)]
MLA_CONFIGS = [(2, 1), (4, 4), (8, 4)]


def _profiles(rng, sq):
    """Seeded length-set generators: (lens, min_process_len)."""
    k = rng.randrange(6)
    if k == 0:    # a few dozen requests of 2k - 6k keys
        return [rng.randint(2000, 6000) for _ in range(rng.randint(12, 40))], 64
    if k == 1:    # one long request: bins of one row
        return [rng.randint(12000, 40000)], 64
    if k == 2:    # many short requests: bins of many rows
        return [rng.randint(sq, 128) for _ in range(2048)], 64
    if k == 3:    # a large min_process_len: a short last bin
        return [rng.randint(sq, 6000) for _ in range(rng.randint(2, 24))], rng.choice([1024, 4096])
    if k == 4:    # MTP tails: the last chunk shorter than sq keys
        return [128 * rng.randint(2, 40) + rng.randint(1, max(1, sq - 1))
                for _ in range(rng.randint(8, 32))], 64
    return [rng.randint(sq, 4096) for _ in range(rng.randint(1, 48))], rng.choice([64, 512, 1024])


def catalogue(kind, num_ctas, seed=0, tries=240):
    """Seeded search over _profiles: {path: dict(config, lens, mpl, ctas)} for every path of
    PATHS + SUBPATHS reached, keeping per path the case with the fewest keys x heads (the cost
    of its fp64 reference). kind "fp8" (config (hkv, sq, group)) or "mla" (config (T, sq))."""
    rng = random.Random(seed)
    configs = FP8_CONFIGS if kind == "fp8" else MLA_CONFIGS
    want = set(PATHS) | set(SUBPATHS)
    found = {}
    for t in range(tries):
        cfg = configs[t % len(configs)]
        hkv, sq = cfg[0], cfg[1]
        lens, mpl = _profiles(rng, sq)
        cost = sum(lens) * hkv
        tm = task_map(lens, num_ctas, hkv, sq, mpl)
        for p, n in path_counts(walk(tm, len(lens), hkv), sq).items():
            if p in want and (p not in found or cost < found[p]["cost"]):
                found[p] = dict(config=cfg, lens=lens, mpl=mpl, ctas=n, cost=cost)
    return found


# ------------------------------------------------------------------------------------------------
# walk mutations
# ------------------------------------------------------------------------------------------------
def mutation_weights(walks, mutation, num_batch, num_head_kv):
    """{(b, h): (w_num, w_den, keys)} key weights of the pairs a mutation changes (per key of
    the request: y = sum w_num p v / sum w_den p), plus {(b, h): (b', h')} pairs whose rows
    receive another pair's result (restore_wrong_target on a direct write) and a set of pairs
    left unwritten."""
    weights, moved, unwritten = {}, {}, set()

    def w_of(b, h, n):
        if (b, h) not in weights:
            weights[(b, h)] = (np.ones(n), np.ones(n))
        return weights[(b, h)]

    if mutation == "fallback_not_taken":
        for w in walks:
            if w["u0"] > 0 and not w["found"]:
                for s in w["segs"]:
                    n = s["start"] + s["keys"]
                    if s["nchunks"] == 1:
                        unwritten.add((s["b"], s["h"]))
                    else:
                        wn, wd = w_of(s["b"], s["h"], _req_len(walks, s["b"], s["h"]))
                        wn[s["start"]:n] = 0
                        wd[s["start"]:n] = 0
        return weights, moved, unwritten
    for w in walks:
        s = split_task(w)
        if s is None:
            continue
        b, h = s["b"], s["h"]
        n = _req_len(walks, b, h)
        seam, end = s["start"] + w["o"] * TILE, s["start"] + s["keys"]
        if mutation == "none":  # the evaluator itself: every weight 1
            w_of(b, h, n)
            continue
        if mutation == "restore_wrong_target":
            if s["nchunks"] == 1:
                moved[(b, h)] = ((b + 1) % num_batch, h) if num_batch > 1 else (b, (h + 1) % num_head_kv)
            else:  # the partial lands in a neighbouring chunk's slot: that chunk counts twice
                cs = _chunk_ranges(walks, b, h)
                c2 = s["chunk"] + 1 if s["chunk"] + 1 < len(cs) else s["chunk"] - 1
                wn, wd = w_of(b, h, n)
                wn[s["start"]:end] = 0
                wd[s["start"]:end] = 0
                wn[cs[c2][0]:cs[c2][1]] *= 2
                wd[cs[c2][0]:cs[c2][1]] *= 2
            continue
        wn, wd = w_of(b, h, n)
        if mutation == "seam_tile_dropped":
            wn[seam:min(seam + TILE, end)] = 0
            wd[seam:min(seam + TILE, end)] = 0
        elif mutation == "seam_tile_twice":
            wn[seam:min(seam + TILE, end)] *= 2
            wd[seam:min(seam + TILE, end)] *= 2
        elif mutation == "carry_lost":
            wn[seam:end] = 0
            wd[seam:end] = 0
        elif mutation == "l_not_carried":
            wd[seam:end] = 0
        else:
            raise ValueError(mutation)
    return weights, moved, unwritten


def _req_len(walks, b, h):
    return max(s["start"] + s["keys"] for w in walks for s in w["segs"]
               if s["b"] == b and s["h"] == h)


def _chunk_ranges(walks, b, h):
    return [(st, st + n) for st, n in pair_chunks(walks)[(b, h)]]


def weighted_rows(s, v, wn, wd):
    """fp64 y = sum_j wn_j p_j v_j / sum_j wd_j p_j for scores s [R, N] (-inf: masked)."""
    wn = torch.as_tensor(wn[:s.shape[1]], dtype=torch.float64)
    wd = torch.as_tensor(wd[:s.shape[1]], dtype=torch.float64)
    m = s.max(1, keepdim=True).values
    m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
    p = torch.exp(s - m)
    return ((p * wn) @ v) / (p * wd).sum(1, keepdim=True)


def mutant(lossy, walks, mutation, pair_fn, num_batch, num_head_kv):
    """The lossy oracle's output with the rows of every pair `mutation` changes replaced.
    pair_fn(b, h) -> (scores [R, N] float64 with -inf on masked keys, values [N, D] float64,
    output index of its R rows into lossy)."""
    out = lossy.clone().double()
    weights, moved, unwritten = mutation_weights(walks, mutation, num_batch, num_head_kv)
    for (b, h), (wn, wd) in weights.items():
        s, v, idx = pair_fn(b, h)
        out[idx] = weighted_rows(s, v, wn, wd).to(torch.bfloat16).double()
    for (b, h), dst in moved.items():  # pair (b, h)'s result lands on dst's rows, its own stay unwritten
        out[pair_fn(*dst)[2]] = lossy.double()[pair_fn(b, h)[2]]
        unwritten.add((b, h))
    for bh in unwritten:
        out[pair_fn(*bh)[2]] = math.nan
    return out


def fp8_pair_fn(d, num_seq_q, k_per_token):
    """pair_fn of mutant() for a synth.attention_exact decode case: the fp64 scores and values of
    the rows of (request b, kv head h), as oracle.attention_exact.decode_fp8_exact forms them."""
    from oracle.attention_exact import _kpt_scales, _paged
    k = d["kcache"] if k_per_token else d["kvcache"][:, 0]
    v = d["vcache"] if k_per_token else d["kvcache"][:, 1]
    hq, dim = d["q"].shape[1], d["q"].shape[2]
    hkv, bs, sq = k.shape[2], k.shape[1], num_seq_q
    g = hq // hkv
    lens = d["kv_lens_total"].tolist()

    def f(b, h):
        n = lens[b]
        ids = d["block_ids"][b, :(n + bs - 1) // bs]
        kc, vc = _paged(k, ids, n, h), _paged(v, ids, n, h)
        if k_per_token:
            ck, vs, kt = _kpt_scales(d["k_scale"], ids, n, h), float(d["v_scale"][h]), 1.0
        else:
            ck, vs = torch.ones(n, dtype=torch.float64), float(d["v_scale"][0])
            kt = float(d["k_scale"][0])
        gi, i = torch.meshgrid(torch.arange(g), torch.arange(sq), indexing="ij")
        gi, i = gi.reshape(-1), i.reshape(-1)
        rows, heads = b * sq + i, h * g + gi
        qc = d["q"][rows, heads].double()
        cq = d["q_scale"][rows, heads].double() * kt / math.sqrt(dim)
        s = (qc @ kc.T) * cq[:, None] * ck[None, :]
        vis = torch.arange(n)[None, :] <= (n - sq + i)[:, None]
        return torch.where(vis, s, torch.full_like(s, -math.inf)), vc * vs, (rows, heads)
    return f


def mla_pair_fn(d):
    """pair_fn of mutant() for a synth.attention_mla case: rows of (request b, query tile t)."""
    h, sq, scale = d["h"], d["num_seq_q"], d["scale"]
    lens = d["lens_total"].tolist()

    def f(b, t):
        n = lens[b]
        npg = (n + 63) // 64
        k = d["kv"][d["block_ids"][b, :npg].long()].reshape(-1, d["kv"].shape[2])[:n].double()
        ri = torch.arange(64 * t, min(64 * t + 64, sq * h))
        rows, heads = b * sq + ri // h, ri % h
        s = (d["q"][rows, heads].double() @ k.T) * scale
        vis = torch.arange(n)[None, :] <= (n - sq + ri // h)[:, None]
        return torch.where(vis, s, torch.full_like(s, -math.inf)), k[:, :512], (rows, heads)
    return f


def mla_chunk_slot(base, c):
    """decode_attn_mla.cu chunk_slot: the partial slot of chunk c of a pair whose chunk 0 ran in
    bin `base`."""
    return 2 * base + 1 if c == 0 else 2 * (base + c)
