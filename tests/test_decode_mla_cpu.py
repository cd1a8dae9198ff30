"""CPU side of the absorbed MLA decode: the exact oracle and its mutants, the split-partial slot
rule against the scheduler, the C launcher's rejections and the fake op's shape."""
import ctypes
import random

import numpy as np
import pytest
import torch

from oracle import attention_mla as om
from oracle import taskmap
from synth import attention_mla as sm

CASES = [
    # (lengths, H, mtp, kind, scale, min_process_len)
    ([3000, 65, 2, 700, 129], 128, 1, "wide", sm.SCALE_DSV3, 64),
    (sm.lengths(1), 16, 0, "pe", sm.SCALE_PLAIN, 64),
    (sm.lengths(4), 32, 3, "vhigh", sm.SCALE_DSV3, 64),
    ([1500, 63, 64], 64, 1, "wide", sm.SCALE_PLAIN, 64),
    ([900, 5], 8, 3, "pe", sm.SCALE_DSV3, 64),
]


def _cases():
    return [sm.make_case(l, h, m, seed=i, kind=k, scale=s, min_process_len=mpl)
            for i, (l, h, m, k, s, mpl) in enumerate(CASES)]


@pytest.fixture(scope="module")
def cases():
    return _cases()


def test_lossy_oracle_passes_exact_check(cases):
    for d in cases:
        r = om.check(om.mla_exact(d["q"], d["kv"], d["block_ids"], d["lens_total"],
                                  d["num_seq_q"], d["scale"], d["chunks"], lossy=True)[0], d)
        assert r["ok_a"] and r["ok_b"], (d["kind"], d["h"], r)


def test_cases_cover_the_gpu_claims(cases):
    assert {d["h"] for d in cases} == {8, 16, 32, 64, 128}
    assert {d["mtp"] for d in cases} >= {0, 1, 3}
    nch = [len(v) for d in cases for v in d["chunks"].values()]
    assert min(nch) == 1 and max(nch) > 2  # single-chunk and multi-chunk pairs
    assert any(om.num_tiles(d["h"], d["num_seq_q"]) > 1 for d in cases)  # tile boundaries
    assert any(om.num_tiles(d["h"], d["num_seq_q"]) * 64 > d["h"] * d["num_seq_q"] or
               d["h"] < 64 for d in cases)  # a tile holding several tokens


@pytest.mark.parametrize("mutation", om.MUTATIONS)
def test_every_mutation_is_caught(cases, mutation):
    caught = []
    for i, d in enumerate(cases):
        r = om.check(om.mutant(d, mutation), d)
        if not (r["ok_a"] and r["ok_b"]):
            caught.append(i)
    print(f"mutation {mutation}: caught by cases {caught}")
    assert caught, mutation


def test_split_partial_slots_are_unique():
    """Two slots per bin hold every split chunk (decode_attn_mla.cu `chunk_slot`): chunk c > 0
    starts its bin, chunk 0 of a split pair ends its bin. Checked over random schedules."""
    rng = random.Random(1)
    for trial in range(200):
        nb = rng.randint(1, 40)
        h = rng.choice([8, 16, 32, 64, 128])
        sq = rng.randint(1, 4)
        T = om.num_tiles(h, sq)
        ctas = rng.choice([132, 114, 7])
        lens = [rng.choice([rng.randint(sq, 200), rng.randint(sq, 20000)]) for _ in range(nb)]
        tm = taskmap.assign(lens, ctas, T, sq, 128, True, rng.choice([64, 512]))
        ntpc1 = int(tm[0, 0])
        rows = tm[1:1 + ntpc1 * ctas].reshape(ctas, ntpc1, 12)
        chunk_tab = tm[1 + ntpc1 * ctas:].reshape(-1)[:T * nb]
        used = {}
        for icta in range(ctas):
            for r in rows[icta]:
                hh, b, c = int(r[0]), int(r[1]), int(r[2])
                if hh < 0 or b < 0:
                    break
                if chunk_tab[hh * nb + b] <= 1:
                    continue
                base = icta - c
                slot = 2 * base + 1 if c == 0 else 2 * (base + c)
                assert slot not in used, (trial, icta, used.get(slot), (hh, b, c))
                assert 0 <= slot < 2 * ctas
                used[slot] = (hh, b, c)
        assert len(used) <= 2 * ctas


def _lib(hpc):
    return hpc._ffi.lib


def test_launcher_rejections(hpc):
    lib = _lib(hpc)
    P = ctypes.c_void_p(1 << 20)
    I = ctypes.cast(P, ctypes.POINTER(ctypes.c_int))

    def call(**kw):
        a = dict(num_batch=2, num_seq_q=1, num_head_q=16, num_dim_qk=576, num_kvcache_blocks=4,
                 block_size=64, num_seq_max_blocks=2, ldY=16 * 512, ldQ=16 * 576,
                 kv_block_stride=64 * 576, kv_token_stride=576, scale=0.1, ctas=132)
        a.update(kw)
        return lib.hpc_attention_decode_mla_bf16_async(
            P, P, I, I, P, P, I, a["num_batch"], a["num_seq_q"], a["num_head_q"], a["num_dim_qk"],
            a["num_kvcache_blocks"], a["block_size"], a["num_seq_max_blocks"], a["ldY"], a["ldQ"],
            a["kv_block_stride"], a["kv_token_stride"], a["scale"], a["ctas"], None)

    for bad in (dict(num_head_q=12), dict(num_head_q=256), dict(num_seq_q=5), dict(num_seq_q=0),
                dict(num_dim_qk=512), dict(block_size=32), dict(num_batch=2049),
                dict(kv_token_stride=580), dict(kv_token_stride=568), dict(kv_block_stride=36868),
                dict(ldQ=16 * 576 + 4), dict(ldY=16 * 512 + 2)):
        assert call(**bad) == 1, bad
        assert hpc._ffi.lib.hpc_last_error()


def test_fake_shape(hpc):
    from hpc.attention import _attention_decode_mla_bf16_fake as fake
    q = torch.empty(6, 32, 576, dtype=torch.bfloat16, device="meta")
    kv = torch.empty(10, 64, 576, dtype=torch.bfloat16, device="meta")
    ids = torch.empty(3, 4, dtype=torch.int32, device="meta")
    lens = torch.empty(3, dtype=torch.int32, device="meta")
    y = fake(q, kv, ids, lens, 0.1, 1, False, None, None)
    assert y.shape == (6, 32, 512) and y.dtype == torch.bfloat16
    out = torch.empty(6, 32, 512, dtype=torch.bfloat16, device="meta")
    assert fake(q, kv, ids, lens, 0.1, 1, False, None, out) is out
    assert hasattr(torch.ops.hpc, "attention_decode_mla_bf16")
    assert hpc.mla_num_query_tiles(128, 1) == 4 and hpc.mla_num_query_tiles(8, 0) == 1
