"""The rotated bin walk of the FP8 and MLA decode kernels (csrc/decode_common.cuh), restated in
oracle/decode_walk.py, without a GPU: hand-built bins pin the restatement to the device code,
properties hold over many seeded task maps, a seeded search reaches every walk path at 132 and
114 CTAs, and every walk bug of decode_walk.MUTATIONS fails the exact check on seam-aware inputs
(synth/attention_exact.py, synth/attention_mla.py)."""
import random

import numpy as np
import pytest
import torch

from oracle import attention_exact as ox
from oracle import attention_mla as om
from oracle import decode_walk as dw
from synth import attention_mla as sm
from synth.attention_exact import make_decode_exact_inputs
from test_attention_exact_cpu import decode_exact, decode_lossy


def _bin(tiles, rows=None):
    """A bin of task rows with the given tile counts, terminated (rows: max_rows + 1)."""
    rows = rows or len(tiles) + 1
    b = np.zeros((rows, dw.ROW), dtype=np.int32)
    b[:, :2] = -1
    for i, t in enumerate(tiles):
        b[i, :2] = (0, i)
        b[i, 6] = t
    return b


# ------------------------------------------------------------------------------------------------
# hand-built bins with known answers
# ------------------------------------------------------------------------------------------------
def test_scan_bin_known_answers():
    # u0 == 0: front to back, rows read until the terminator
    assert dw.scan_bin(_bin([5, 3, 4], 8), 7, 0) == (7, 0, 0, False)
    # hit in row 0: its tail [2, 5) first, head [0, 2) last
    assert dw.scan_bin(_bin([5, 3, 4], 8), 7, 2) == (3, 0, 2, True)
    # hit at a task boundary: row 1 from its first tile
    assert dw.scan_bin(_bin([5, 3, 4], 8), 7, 5) == (3, 1, 0, True)
    # second ballot round: 40 rows of one tile, u0 = 35 -> row 35; 3-tile rows: u0 = 100 -> row 33
    assert dw.scan_bin(_bin([1] * 40, 64), 63, 35) == (40, 35, 0, True)
    assert dw.scan_bin(_bin([3] * 40, 64), 63, 100) == (40, 33, 1, True)
    # exactly 32 rows, then the terminator in the next round
    assert dw.scan_bin(_bin([1] * 32, 40), 39, 31) == (32, 31, 0, True)
    # u0 past the last tile: the short-bin fallback
    assert dw.scan_bin(_bin([2, 2], 8), 7, 7) == (2, 0, 0, False)
    assert dw.scan_bin(_bin([2, 2], 8), 7, 4) == (2, 0, 0, False)
    # an empty bin
    assert dw.scan_bin(_bin([], 8), 7, 3) == (0, 0, 0, False)


def test_segment_order_known_answer():
    segs = [dw.segment_of(3, 1, 2, j) for j in range(4)]
    assert [(s["row"], s["tb"], s["te"], s["save"], s["restore"]) for s in segs] == [
        (1, 2, -1, True, False), (2, 0, -1, False, False), (0, 0, -1, False, False),
        (1, 0, 2, False, True)]
    # a single-row bin: its own tail, then its own head
    assert [(s["row"], s["tb"], s["te"]) for s in (dw.segment_of(1, 0, 3, 0),
                                                  dw.segment_of(1, 0, 3, 1))] == [(0, 3, -1), (0, 0, 3)]


def test_walk_start_known_answers():
    tm = np.zeros((1, dw.ROW), dtype=np.int32)
    tm[0, 0], tm[0, 6] = 11, 35  # P = 10, TB = 35
    assert [dw.walk_start(tm, i) for i in range(5)] == [0, 0, 0, 0, 5]  # x0 = 40: 40 % 35 = 5
    assert dw.walk_start(tm, 6) == 5                                      # 60 % 35 = 25 -> 5
    tm[0, 6] = 0  # a map without TB is walked front to back
    assert dw.walk_start(tm, 4) == 0


def test_scan_bin_equals_a_plain_prefix_search():
    rng = random.Random(3)
    for _ in range(400):
        n = rng.randint(0, 80)
        tiles = [rng.randint(1, 5) for _ in range(n)]
        P = max(sum(tiles), n, 1)
        u0 = rng.randint(0, P + 3)
        m, ks, o, found = dw.scan_bin(_bin(tiles, P + 1), P, u0)
        if u0 == 0:
            assert (m, ks, o, found) == (P, 0, 0, False)
            continue
        cum = np.cumsum([0] + tiles)
        hit = [i for i in range(n) if cum[i] <= u0 < cum[i + 1]]
        assert m == n
        assert (ks, o, found) == ((hit[0], u0 - int(cum[hit[0]]), True) if hit else (0, 0, False))


# ------------------------------------------------------------------------------------------------
# properties over seeded task maps
# ------------------------------------------------------------------------------------------------
def _random_maps(seed, count):
    rng = random.Random(seed)
    for _ in range(count):
        nb = rng.choice([1, 2, 7, 40, 300, 2048])
        mla = rng.random() < 0.4
        hkv = rng.choice([2, 4, 8]) if mla else rng.choice([1, 2, 4, 6, 8])
        sq = rng.randint(1, 4)
        mpl = rng.choice([64, 128, 512, 1024, 4096])
        ctas = rng.choice([132, 114])
        top = rng.choice([130, 3000, 40000]) if nb <= 40 else rng.choice([130, 600])
        lens = [rng.randint(sq, top) for _ in range(nb)]
        yield lens, ctas, hkv, sq, mpl, mla


def test_walk_properties_over_seeded_maps():
    n_split = n_rows = 0
    for lens, ctas, hkv, sq, mpl, mla in _random_maps(7, 60):
        tag = (len(lens), ctas, hkv, sq, mpl)
        tm = dw.task_map(lens, ctas, hkv, sq, mpl)
        nb = len(lens)
        walks = dw.walk(tm, nb, hkv)
        ntpc1 = int(tm[0, 0])
        # every tile of every task exactly once
        vis = dw.visits(walks)
        rows = tm[1:1 + ntpc1 * ctas]
        tasks = {(int(r[1]), int(r[0]), int(r[2])): int(r[6]) for r in rows if r[0] >= 0 and r[1] >= 0}
        assert set(vis) == set(tasks), tag
        for key, n in tasks.items():
            assert sorted(vis[key]) == list(range(n)), (tag, key)
        slots = {}
        for icta, w in enumerate(walks):
            segs = w["segs"]
            saves = [j for j, s in enumerate(segs) if s["save"]]
            restores = [j for j, s in enumerate(segs) if s["restore"]]
            assert len(saves) == len(restores) <= 1, tag
            if saves:
                n_split += 1
                n_rows += w["m"]
                a, z = segs[saves[0]], segs[restores[0]]
                assert saves == [0] and restores == [len(segs) - 1], tag  # restore comes last
                assert (a["b"], a["h"], a["chunk"], a["row"]) == (z["b"], z["h"], z["chunk"], z["row"])
                assert (a["tb"], a["te"], z["tb"], z["te"]) == (w["o"], -1, 0, w["o"]), tag
                assert 0 < w["o"] < a["tiles"], tag
                assert "d:middle" not in dw.labels(w, sq), tag  # a middle chunk fills its bin
            if mla:  # MLA's chunk_slot: no two split chunks share a partial slot
                for s in segs:
                    if s["write"] == "split":
                        slot = dw.mla_chunk_slot(icta - s["chunk"], s["chunk"])
                        assert slot not in slots and 0 <= slot < 2 * ctas, (tag, slot)
                        slots[slot] = (s["b"], s["h"], s["chunk"])
        # TB: the splice formula of hpc/attention.py equals the tiles of one head on the line
        assert int(tm[0, 6]) == sum(n for (b, h, c), n in tasks.items() if h == 0), tag
        assert int(tm[0, 6]) == dw.header_tiles(np.asarray(lens) - sq, sq, new_kv_included=False)
    assert n_split > 100 and n_rows > n_split  # the maps do split walks, multi-row ones included


def test_splice_matches_the_oracle_header(hpc, monkeypatch):
    """hpc.assign_attention_decode_task on CPU lengths: the host scheduler's rows and the header
    int 6 it splices equal oracle.decode_walk.task_map (which restates the device scheduler's
    tot_tiles)."""
    import hpc.attention as ha
    rng = random.Random(5)
    for ctas in (132, 114):
        monkeypatch.setattr(ha, "_num_total_ctas", lambda device=None: ctas)
        for _ in range(6):
            sq = rng.randint(1, 4)
            lens = [rng.randint(sq, 9000) for _ in range(rng.randint(1, 64))]
            hkv, mpl, nkv = rng.choice([2, 4, 8]), rng.choice([64, 512]), rng.random() < 0.5
            want = dw.task_map(lens, ctas, hkv, sq, mpl, nkv)
            tm = torch.zeros(want.size * 4 + 4096, dtype=torch.int8)
            hpc.assign_attention_decode_task(torch.tensor(lens, dtype=torch.int32), tm, hkv, sq,
                                             nkv, mpl)
            got = tm[:want.size * 4].view(torch.int32).reshape(-1, dw.ROW).numpy()
            assert int(got[0, 6]) == int(want[0, 6])
            assert np.array_equal(got[1:], want[1:])


# ------------------------------------------------------------------------------------------------
# the path catalogue
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ctas", [132, 114])
@pytest.mark.parametrize("kind", ["fp8", "mla"])
def test_path_catalogue_reaches_every_path(kind, ctas):
    cat = dw.catalogue(kind, ctas)
    for p in dw.PATHS + dw.SUBPATHS:
        if p in cat:
            e = cat[p]
            print(f"CATALOGUE {kind} ctas={ctas} path {p}: config {e['config']} B={len(e['lens'])} "
                  f"keys={sum(e['lens'])} mpl={e['mpl']} CTAs on the path: {e['ctas']}")
    missing = [p for p in dw.PATHS + dw.SUBPATHS if p not in cat]
    assert not missing, missing


def test_c2_path_counts():
    """The C2 benchmark shape (B = 64, 8 kv heads, 8192 keys, sq 1, min_process_len 64) and the
    in-call schedule (min_process_len 512): how many CTAs take each path."""
    for ctas in (132, 114):
        for mpl in (64, 512):
            walks = dw.walk(dw.task_map([8192] * 64, ctas, 8, 1, mpl), 64, 8)
            cnt = dw.path_counts(walks, 1)
            print(f"C2 ctas={ctas} mpl={mpl}: " + " ".join(f"{p}={cnt.get(p, 0)}"
                                                          for p in dw.PATHS + dw.SUBPATHS))
            assert cnt.get("d:only", 0) > 0  # split single-chunk pairs written after the restore


# ------------------------------------------------------------------------------------------------
# walk mutations against the exact check
# ------------------------------------------------------------------------------------------------
CTAS = 132
_CAT = {}


def _cat(kind):
    if kind not in _CAT:
        _CAT[kind] = dw.catalogue(kind, CTAS)
    return _CAT[kind]


def _fp8_case(path, kpt, climb):
    e = _cat("fp8")[path]
    hkv, sq, g = e["config"]
    walks = dw.walk(dw.task_map(e["lens"], CTAS, hkv, sq, e["mpl"]), len(e["lens"]), hkv)
    d = make_decode_exact_inputs("needle", e["lens"], sq, hkv, hkv * g, k_per_token=kpt, seed=31,
                                 seams=dw.seam_keys(walks), heads=dw.head_ranges(walks),
                                 climb=climb)
    if kpt:
        kv = d["kvcache"]
        d.update(kcache=kv[:, 0, :64], vcache=kv[:, 1, :64], k_scale=kv[:, 0, 64:])
    y, bound = decode_exact(d, sq, kpt)
    lossy = decode_lossy(d, sq, kpt)
    return walks, y, bound, lossy, dw.fp8_pair_fn(d, sq, kpt), len(e["lens"]), hkv


def _mla_case(path, climb):
    e = _cat("mla")[path]
    T, sq = e["config"]
    h = {(2, 1): 128, (4, 4): 64, (8, 4): 128}[(T, sq)]
    walks = dw.walk(dw.task_map(e["lens"], CTAS, T, sq, e["mpl"]), len(e["lens"]), T)
    d = sm.make_case(e["lens"], h, sq - 1, seed=32, kind="needle", num_total_ctas=CTAS,
                     min_process_len=e["mpl"], seams=dw.seam_keys(walks),
                     heads=dw.head_ranges(walks), climb=climb)
    args = (d["q"], d["kv"], d["block_ids"], d["lens_total"], sq, d["scale"], d["chunks"])
    y, bound = om.mla_exact(*args)
    lossy = om.mla_exact(*args, lossy=True)[0]
    return walks, y, bound, lossy, dw.mla_pair_fn(d), len(e["lens"]), T


MUTATION_CASES = [("fp8", "d:only", False, 4.0), ("fp8", "d:first", True, -4.0),
                  ("fp8", "g", False, 0.0), ("mla", "d:last", None, 4.0),
                  ("mla", "g", None, -4.0)]


@pytest.fixture(scope="module")
def mutation_cases():
    out = []
    for kind, path, kpt, climb in MUTATION_CASES:
        c = _fp8_case(path, kpt, climb) if kind == "fp8" else _mla_case(path, climb)
        out.append((f"{kind} {path} climb{climb}", c))
    return out


def test_lossy_and_identity_pass_the_exact_check(mutation_cases):
    for tag, (walks, y, bound, lossy, fn, nb, nh) in mutation_cases:
        r = ox.grade(lossy, y, bound, lossy)
        assert r["ok_a"] and r["ok_b"], (tag, r)
        r = ox.grade(dw.mutant(lossy, walks, "none", fn, nb, nh), y, bound, lossy)
        assert r["ok_a"] and r["ok_b"], (tag, "identity", r)


@pytest.mark.parametrize("mutation", dw.MUTATIONS)
def test_every_walk_mutation_is_caught(mutation_cases, mutation):
    caught = []
    for tag, (walks, y, bound, lossy, fn, nb, nh) in mutation_cases:
        m = dw.mutant(lossy, walks, mutation, fn, nb, nh)
        r = ox.grade(m, y, bound, lossy)
        if not (r["ok_a"] and r["ok_b"] and r["nan_ok"]):
            caught.append(tag)
    print(f"walk mutation {mutation}: caught by {caught}")
    assert caught, mutation
