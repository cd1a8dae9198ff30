"""The rotated bin walk of the FP8 and MLA decode kernels on the GPU: one case per walk path of
oracle/decode_walk.py (found by its seeded search on the device's own CTA count), needles on
both sides of every seam (synth/attention_exact.py, synth/attention_mla.py), graded with the
exact two-part check. Before grading, every case asserts from the walk model that the call takes
the path it is named after; it fails rather than skips when it does not. Each run prints one
`EXACT <path tags> ...` line (visible with -s)."""
import pytest
import torch

from oracle import attention_exact as ox
from oracle import attention_mla as om
from oracle import decode_walk as dw
from synth import attention_mla as sm
from synth.attention_exact import make_decode_exact_inputs
from test_attention_exact_cpu import decode_exact, decode_lossy

pytestmark = pytest.mark.gpu

MLA_HEADS = {(2, 1): 128, (4, 4): 64, (8, 4): 128}  # (T, sq) -> H: h128/mtp0, h64/mtp3, h128/mtp3
_CAT = {}


def _ctas(hpc):
    return hpc._ffi.sm_count(torch.device("cuda", 0))


def _catalogue(kind, ctas):
    if (kind, ctas) not in _CAT:
        _CAT[(kind, ctas)] = dw.catalogue(kind, ctas)
    return _CAT[(kind, ctas)]


def _cases(kind, ctas):
    """Distinct catalogue cases: [(paths, entry)]; every path and sub-path is required."""
    cat = _catalogue(kind, ctas)
    missing = [p for p in dw.PATHS + dw.SUBPATHS if p not in cat]
    assert not missing, f"{kind}: no case reaches {missing} on {ctas} CTAs"
    out = {}
    for p in dw.PATHS + dw.SUBPATHS:
        e = cat[p]
        key = (e["config"], tuple(e["lens"]), e["mpl"])
        out.setdefault(key, ([], e))[0].append(p)
    return list(out.values())


def _walks(lens, ctas, hkv, sq, mpl, rotate=True):
    return dw.walk(dw.task_map(lens, ctas, hkv, sq, mpl), len(lens), hkv, rotate=rotate)


def _require(walks, sq, paths, tag):
    cnt = dw.path_counts(walks, sq)
    missing = [p for p in paths if not cnt.get(p)]
    assert not missing, f"{tag}: the walk model says this call does not take {missing}: {cnt}"
    return cnt


# ------------------------------------------------------------------------------------------------
# FP8
# ------------------------------------------------------------------------------------------------
def _fp8_inputs(lens, sq, hkv, g, kpt, walks, climb, seed, layout="NHD"):
    return make_decode_exact_inputs("needle", lens, sq, hkv, hkv * g, k_per_token=kpt,
                                    layout=layout, seed=seed, seams=dw.seam_keys(walks),
                                    heads=dw.head_ranges(walks), climb=climb)


def _fp8_run(hpc, d, sq, kpt, mpl, src="gpu"):
    kv = d["kvcache"].cuda()
    lens = d["kv_lens_total"].cuda()
    hkv = kv.shape[3]
    tm = None
    if src != "none":
        tm = hpc.get_attention_decode_task_workspace(lens.numel(), int(lens.max()), hkv, mpl)
        hpc.assign_attention_decode_task(lens.cpu() if src == "cpu" else lens, tm, hkv, sq, True,
                                         mpl)
        if src == "int6_zero":  # a map without TB: the kernel walks every bin front to back
            tm.view(torch.int32)[6] = 0
    if kpt:
        k, v, ks = kv[:, 0, :64], kv[:, 1, :64], kv[:, 0, 64:]
        qt = hpc.QuantType.QPERTOKEN_PERHEAD_KPERTOKEN_PERHEAD_VPERHEAD
    else:
        k, v, ks = kv[:, 0], kv[:, 1], d["k_scale"].cuda()
        qt = hpc.QuantType.QPERTOKEN_PERHEAD_KPERTENSOR_VPERTENSOR
    y = hpc.attention_decode_fp8(d["q"].cuda(), k, v, d["block_ids"].cuda(), lens,
                                 d["q_scale"].cuda(), ks, d["v_scale"].cuda(), mtp=sq - 1,
                                 new_kv_included=True, quant_type=qt, splitk=True, task_map=tm)
    return y.cpu()


def _report(tag, out, exact, bound, lossy):
    r = ox.assert_exact(out, exact, bound, lossy, tag)
    print(f"EXACT {tag} worst={r['worst']:.4f} rel={r['rel']:.3e} rel_oracle={r['rel_oracle']:.3e}")


def _fp8_grade(hpc, tag, d, sq, kpt, runs):
    """runs: [(min_process_len, map source)]."""
    exact, bound = decode_exact(d, sq, kpt)
    lossy = decode_lossy(d, sq, kpt)
    for mpl, src in runs:
        _report(f"{tag} mpl{mpl} map={src}", _fp8_run(hpc, d, sq, kpt, mpl, src), exact, bound,
                lossy)


@pytest.mark.parametrize("kpt", [False, True])
def test_fp8_every_walk_path(hpc, kpt):
    ctas = _ctas(hpc)
    for i, (paths, e) in enumerate(_cases("fp8", ctas)):
        (hkv, sq, g), lens, mpl = e["config"], e["lens"], e["mpl"]
        walks = _walks(lens, ctas, hkv, sq, mpl)
        cnt = _require(walks, sq, paths, f"fp8 {paths}")
        climb = (4.0, -4.0, 0.0)[i % 3]
        d = _fp8_inputs(lens, sq, hkv, g, kpt, walks, climb, seed=40 + i)
        tag = (f"fp8 paths={'/'.join(paths)} kpt={kpt} hkv{hkv} sq{sq} g{g} B{len(lens)} "
               f"climb{climb} ctas_on_path={[cnt[p] for p in paths]}")
        _fp8_grade(hpc, tag, d, sq, kpt, [(mpl, "gpu")])


@pytest.mark.parametrize("kpt", [False, True])
def test_fp8_map_sources_and_hnd_control(hpc, kpt):
    """One multi-row split case from every task-map source (the GPU scheduler, a CPU map spliced
    in, the in-call schedule, a map with int 6 zeroed: front to back), and the same data in an
    HND cache, which the kernel never rotates."""
    ctas = _ctas(hpc)
    e = _catalogue("fp8", ctas)["d:only"]
    (hkv, sq, g), lens, mpl = e["config"], e["lens"], e["mpl"]
    walks = _walks(lens, ctas, hkv, sq, mpl)
    _require(walks, sq, ["d", "d:only"], "fp8 map sources")
    _require(_walks(lens, ctas, hkv, sq, mpl, rotate=False), sq, ["a"], "fp8 int6 zeroed")
    d = _fp8_inputs(lens, sq, hkv, g, kpt, walks, 4.0, seed=61)
    _fp8_grade(hpc, f"fp8 paths=d/d:only kpt={kpt} NHD", d, sq, kpt,
               [(mpl, "gpu"), (mpl, "cpu"), (mpl, "int6_zero"), (512, "none")])
    h = _fp8_inputs(lens, sq, hkv, g, kpt, walks, 4.0, seed=61, layout="HND")
    assert torch.equal(h["kvcache"].view(torch.uint8), d["kvcache"].view(torch.uint8))
    _fp8_grade(hpc, f"fp8 paths=a (HND control) kpt={kpt}", h, sq, kpt, [(mpl, "gpu")])


def _c2_inputs(walks, graded, kpt, seed):
    """C2 (B = 64, GQA 32/8, 8192 keys): needle inputs for the `graded` requests; every other
    request reads copies of their pages (its output is not graded)."""
    B, S, hkv, hq, P = 64, 8192, 8, 32, 8192 // 64
    idx = {b: i for i, b in enumerate(graded)}
    seams = {(idx[b], h): v for (b, h), v in dw.seam_keys(walks).items() if b in idx}
    heads = {(idx[b], h): v for (b, h), v in dw.head_ranges(walks).items() if b in idx}
    sub = make_decode_exact_inputs("needle", [S] * len(graded), 1, hkv, hq, k_per_token=kpt,
                                   seed=seed, seams=seams, heads=heads, climb=4.0)
    nsub = sub["kvcache"].shape[0]
    fill = torch.arange((B - len(graded)) * P) % nsub
    kv = torch.cat([sub["kvcache"], sub["kvcache"][fill]])
    ids = torch.empty(B, P, dtype=torch.int32)
    q = torch.empty(B, hq, 128, dtype=torch.float8_e4m3fn)
    qs = torch.empty(B, hq, dtype=torch.float32)
    o = nsub
    for b in range(B):
        i = idx.get(b, 0)
        q[b], qs[b] = sub["q"][i], sub["q_scale"][i]
        if b in idx:
            ids[b] = sub["block_ids"][i, :P]
        else:
            ids[b] = torch.arange(o, o + P, dtype=torch.int32)
            o += P
    full = dict(sub, q=q, q_scale=qs, kvcache=kv, block_ids=ids,
                kv_lens_total=torch.full((B,), S, dtype=torch.int32))
    return full, sub


@pytest.mark.parametrize("kpt", [False, True])
def test_fp8_c2_full_size_split_requests(hpc, kpt):
    """The C2 schedule at full size: the requests whose tasks the walk model says are split,
    sampled so that every split role of the shape is graded exactly."""
    ctas, mpl = _ctas(hpc), 64
    walks = _walks([8192] * 64, ctas, 8, 1, mpl)
    cnt = _require(walks, 1, ["d", "d:only"], "fp8 C2")
    by_label = {}
    for w in walks:
        s = dw.split_task(w)
        if s is not None:
            for p in sorted(dw.labels(w, 1)):
                by_label.setdefault(p, []).append(s["b"])
    graded = []
    for p in sorted(by_label):
        for b in by_label[p][:2]:
            if b not in graded and len(graded) < 6:
                graded.append(b)
    full, sub = _c2_inputs(walks, graded, kpt, seed=71)
    out = _fp8_run(hpc, full, 1, kpt, mpl)
    exact, bound = decode_exact(sub, 1, kpt)
    lossy = decode_lossy(sub, 1, kpt)
    _report(f"fp8 C2 paths={'/'.join(p for p in dw.PATHS + dw.SUBPATHS if cnt.get(p))} kpt={kpt} "
            f"requests={graded} ctas_on_path={cnt}", out[graded], exact, bound, lossy)


# ------------------------------------------------------------------------------------------------
# MLA
# ------------------------------------------------------------------------------------------------
def _mla_run(hpc, d, T, src="gpu"):
    lens = d["lens_total"].cuda()
    ids = d["block_ids"].cuda()
    sq = d["num_seq_q"]
    tm = hpc.get_attention_decode_task_workspace(len(lens), int(ids.size(1)) * 64 + sq, T,
                                                 d["min_process_len"], device="cuda")
    hpc.assign_attention_decode_task(lens if src == "gpu" else lens.cpu(), tm, T, sq, True,
                                     d["min_process_len"])
    y = hpc.attention_decode_mla_bf16(d["q"].cuda(), d["kv"].cuda(), ids, lens, d["scale"],
                                      mtp=d["mtp"], new_kv_included=True, task_map=tm)
    return y.float().cpu()


def _mla_check(y, d, tag):
    r = om.check(y, d, tag)
    print(f"EXACT {tag} worst={r['worst']:.4f} rel={r['rel']:.3e} rel_oracle={r['rel_oracle']:.3e}")
    assert r["nan_ok"] and r["ok_a"] and r["ok_b"], (tag, r)


def _mla_case(lens, T, sq, mpl, ctas, walks, climb, seed):
    return sm.make_case(lens, MLA_HEADS[(T, sq)], sq - 1, seed=seed, kind="needle",
                        num_total_ctas=ctas, min_process_len=mpl, seams=dw.seam_keys(walks),
                        heads=dw.head_ranges(walks), climb=climb)


def test_mla_every_walk_path(hpc):
    ctas = _ctas(hpc)
    for i, (paths, e) in enumerate(_cases("mla", ctas)):
        (T, sq), lens, mpl = e["config"], e["lens"], e["mpl"]
        walks = _walks(lens, ctas, T, sq, mpl)
        cnt = _require(walks, sq, paths, f"mla {paths}")
        climb = (4.0, -4.0)[i % 2]
        d = _mla_case(lens, T, sq, mpl, ctas, walks, climb, seed=80 + i)
        _mla_check(_mla_run(hpc, d, T), d, f"mla paths={'/'.join(paths)} T{T} sq{sq} "
                   f"B{len(lens)} mpl{mpl} climb{climb} ctas_on_path={[cnt[p] for p in paths]}")


@pytest.mark.parametrize("T,sq", sorted(MLA_HEADS))
def test_mla_multi_row_splits(hpc, T, sq):
    """A few dozen requests of 2k - 6k keys at min_process_len 64: multi-row split bins for
    every T, from the GPU scheduler and from a CPU map spliced in."""
    ctas = _ctas(hpc)
    g = torch.Generator().manual_seed(T * 10 + sq)
    lens = torch.randint(2000, 6001, (24,), generator=g).tolist()
    walks = _walks(lens, ctas, T, sq, 64)
    cnt = _require(walks, sq, ["d"], f"mla T{T}")
    d = _mla_case(lens, T, sq, 64, ctas, walks, 4.0 if T != 4 else -4.0, seed=90 + T)
    for src in ("gpu", "cpu"):
        _mla_check(_mla_run(hpc, d, T, src), d, f"mla paths=d T{T} sq{sq} B24 mpl64 map={src} "
                   f"ctas_on_path={cnt}")


def test_mla_many_short_requests_wide_bins(hpc):
    """2048 short requests at T = 4: bins of more than 32 rows, start rows past 32."""
    ctas = _ctas(hpc)
    g = torch.Generator().manual_seed(12)
    lens = torch.randint(4, 129, (2048,), generator=g).tolist()
    walks = _walks(lens, ctas, 4, 4, 64)
    cnt = _require(walks, 4, ["f"], "mla 2048 short")
    d = _mla_case(lens, 4, 4, 64, ctas, walks, 0.0, seed=13)
    _mla_check(_mla_run(hpc, d, 4), d, f"mla paths=f T4 sq4 B2048 ctas_on_path={cnt}")


def test_mla_graph_replay_carry_does_not_leak(hpc):
    """Capture on lengths whose walks never split, replay on lengths with multi-row splits (the
    carry buffer in use), then on the first lengths again."""
    ctas, T, sq, B, mpl = _ctas(hpc), 2, 1, 24, 64
    g = torch.Generator().manual_seed(14)
    lens1 = [64] * B
    lens2 = torch.randint(2000, 6001, (B,), generator=g).tolist()
    w1, w2 = _walks(lens1, ctas, T, sq, mpl), _walks(lens2, ctas, T, sq, mpl)
    c1 = dw.path_counts(w1, sq)
    assert not (c1.get("c") or c1.get("d")), c1
    c2 = _require(w2, sq, ["d"], "mla graph")
    d1 = _mla_case(lens1, T, sq, mpl, ctas, w1, 0.0, seed=15)
    d2 = _mla_case(lens2, T, sq, mpl, ctas, w2, 4.0, seed=16)
    nblk = max(d1["kv"].size(0), d2["kv"].size(0))
    mb = max(d1["block_ids"].size(1), d2["block_ids"].size(1))
    kv = torch.zeros(nblk, 64, 576, dtype=torch.bfloat16, device="cuda")
    ids = torch.zeros(B, mb, dtype=torch.int32, device="cuda")
    q = torch.zeros_like(d1["q"], device="cuda")
    lens = torch.zeros(B, dtype=torch.int32, device="cuda")
    tm = hpc.get_attention_decode_task_workspace(B, mb * 64 + sq, T, mpl, device="cuda")

    def load(d):
        kv.fill_(float("nan"))
        kv[:d["kv"].size(0)] = d["kv"].cuda()
        ids.zero_()
        ids[:, :d["block_ids"].size(1)] = d["block_ids"].cuda()
        q.copy_(d["q"].cuda())
        lens.copy_(d["lens_total"].cuda())

    def call():
        hpc.assign_attention_decode_task(lens, tm, T, sq, True, mpl)
        return hpc.attention_decode_mla_bf16(q, kv, ids, lens, d1["scale"], mtp=0,
                                             new_kv_included=True, task_map=tm)

    load(d1)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = call()
    for d, tag in ((d1, f"no split {c1}"), (d2, f"multi-row split {c2}"), (d1, "no split again")):
        load(d)
        graph.replay()
        torch.cuda.synchronize()
        _mla_check(y.float().cpu(), d, f"mla paths=graph replay T{T}: {tag}")
