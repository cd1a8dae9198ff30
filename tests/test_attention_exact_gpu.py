"""FP8 attention kernels against the exact fp64 reference (oracle/attention_exact.py), on inputs
whose outputs depend visibly on the scores (synth/attention_exact.py).

Each case passes (a) |kernel - exact| <= B element-wise and (b) rel L2 of the kernel's error
<= AGG_C times the lossy oracle's + AGG_FLOOR. Each case prints one line `EXACT <tag> worst=...
rel=... rel_oracle=...` (visible with -s).
"""
import pytest
import torch

from oracle import attention_exact as ox
from synth.attention_exact import make_decode_exact_inputs, make_prefill_exact_inputs
from test_attention_exact_cpu import decode_exact, decode_lossy, prefill_exact, prefill_lossy

pytestmark = pytest.mark.gpu


def _report(tag, out, y, bound, lossy):
    r = ox.assert_exact(out, y, bound, lossy, tag)
    print(f"EXACT {tag} worst={r['worst']:.4f} rel={r['rel']:.3e} rel_oracle={r['rel_oracle']:.3e}")


# ------------------------------------------------------------------------------------------------
# decode
# ------------------------------------------------------------------------------------------------
def _decode(hpc, d, sq, kpt, mpl=1024, task_map="gpu"):
    c = {k: v.cuda() for k, v in d.items()}
    lens = c["kv_lens_total"]
    hkv = c["kvcache"].shape[3]
    tm = None
    if task_map is not None:
        tm = hpc.get_attention_decode_task_workspace(lens.numel(), int(lens.max()), hkv, mpl)
        hpc.assign_attention_decode_task(lens.cpu() if task_map == "cpu" else lens, tm, hkv, sq,
                                         True, mpl)
    if kpt:
        kv = c["kvcache"]
        k, v, ks = kv[:, 0, :64], kv[:, 1, :64], kv[:, 0, 64:]
        qt = hpc.QuantType.QPERTOKEN_PERHEAD_KPERTOKEN_PERHEAD_VPERHEAD
    else:
        k, v, ks = c["kvcache"][:, 0], c["kvcache"][:, 1], c["k_scale"]
        qt = hpc.QuantType.QPERTOKEN_PERHEAD_KPERTENSOR_VPERTENSOR
    return hpc.attention_decode_fp8(c["q"], k, v, c["block_ids"], lens, c["q_scale"], ks,
                                    c["v_scale"], mtp=sq - 1, new_kv_included=True, quant_type=qt,
                                    splitk=True, task_map=tm).cpu()


def _decode_case(hpc, tag, d, sq, kpt, runs):
    y, bound = decode_exact(d, sq, kpt)
    lossy = decode_lossy(d, sq, kpt)
    for mpl, tm in runs:
        _report(f"{tag} mpl{mpl} tm={tm}", _decode(hpc, d, sq, kpt, mpl, tm), y, bound, lossy)


@pytest.mark.parametrize("kpt", [False, True])
@pytest.mark.parametrize("layout", ["NHD", "HND"])
@pytest.mark.parametrize("sq", [1, 2, 3, 4])
@pytest.mark.parametrize("heads", [(1, 8), (4, 32), (8, 32)])
def test_decode_exact_needles(hpc, kpt, layout, sq, heads):
    lens = [1000 + sq, 131, 77, 2050]
    d = make_decode_exact_inputs("needle", lens, sq, *heads, k_per_token=kpt, layout=layout,
                                 seed=sq)
    _decode_case(hpc, f"decode needle kpt={kpt} {layout} sq{sq} {heads}", d, sq, kpt,
                 [(1024, "gpu")] + ([(64, "gpu"), (64, "cpu"), (1024, None)] if layout == "NHD" else []))


@pytest.mark.parametrize("kpt", [False, True])
@pytest.mark.parametrize("temp", [1.0, 4.0, 16.0])
@pytest.mark.parametrize("layout", ["NHD", "HND"])
def test_decode_exact_peaked(hpc, kpt, temp, layout):
    sq = 2
    lens = [3000, 131, 77, 700, 1]
    lens = [max(n, sq) for n in lens]
    d = make_decode_exact_inputs("peaked", lens, sq, 4, 32, k_per_token=kpt, temperature=temp,
                                 layout=layout, seed=int(temp))
    _decode_case(hpc, f"decode peaked kpt={kpt} T{temp} {layout}", d, sq, kpt,
                 [(64, "gpu"), (1024, "gpu")])


@pytest.mark.parametrize("sq", [1, 2, 4])
@pytest.mark.parametrize("layout", ["NHD", "HND"])
def test_decode_exact_kscale_addressing(hpc, sq, layout):
    lens = [300, 131, 200, 1000]
    d = make_decode_exact_inputs("kscale", lens, sq, 4, 16, k_per_token=True, layout=layout,
                                 seed=11 + sq)
    _decode_case(hpc, f"decode kscale sq{sq} {layout}", d, sq, True, [(64, "gpu"), (1024, None)])


@pytest.mark.parametrize("lens", [[1], [2, 64, 65, 127, 128, 129, 255, 256, 257], [4, 4, 4],
                                  [40000], [129] * 5, [131] * 37])
@pytest.mark.parametrize("sq", [1, 4])
@pytest.mark.parametrize("kpt", [False, True])
def test_decode_exact_edge_lengths(hpc, lens, sq, kpt):
    lens = [max(n, sq) for n in lens]
    d = make_decode_exact_inputs("needle", lens, sq, 2, 8, k_per_token=kpt, seed=7)
    _decode_case(hpc, f"decode edge {lens[:3]} sq{sq} kpt={kpt}", d, sq, kpt,
                 [(64, "gpu"), (1024, "gpu")])


# ------------------------------------------------------------------------------------------------
# prefill
# ------------------------------------------------------------------------------------------------
def _prefill(hpc, d, kpt, dense_api=False):
    c = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in d.items()}
    qt = (hpc.QuantType.QPERTOKEN_PERHEAD_KPERTOKEN_PERHEAD_VPERHEAD if kpt
          else hpc.QuantType.QPERTOKEN_PERHEAD_KPERTENSOR_VPERTENSOR)
    args = (c["q"], c["kcache"], c["vcache"], c["qscale"], c["kscale"], c["vscale"],
            c["cu_seqlens_q"], c["block_ids"], c["seqlens_kv"], d["max_q"])
    if dense_api:
        return hpc.attention_with_kvcache_prefill_fp8(*args, quant_type=qt).cpu()
    mask = c["block_mask"].to(torch.uint8).contiguous() if c["block_mask"] is not None else None
    return hpc.attention_with_kvcache_blocksparse_prefill_fp8(*args, quant_type=qt,
                                                              block_mask=mask).cpu()


def _prefill_case(hpc, tag, d, kpt, dense_api=False):
    y, bound = prefill_exact(d, kpt)
    _report(tag, _prefill(hpc, d, kpt, dense_api), y, bound, prefill_lossy(d, kpt))


@pytest.mark.parametrize("kpt", [False, True])
@pytest.mark.parametrize("seq", [1024, 2048])
@pytest.mark.parametrize("skip", [None, 0.0, 0.5])
@pytest.mark.parametrize("layout", ["nhd", "hnd"])
def test_prefill_exact_reference_grid(hpc, kpt, seq, skip, layout):
    d = make_prefill_exact_inputs([seq, seq], [seq, seq], 4, 1, skip, kpt, kind="peaked",
                                  temperature=4.0, layout=layout, seed=seq)
    _prefill_case(hpc, f"prefill grid kpt={kpt} seq{seq} skip{skip} {layout}", d, kpt)


@pytest.mark.parametrize("kpt", [False, True])
@pytest.mark.parametrize("temp", [1.0, 16.0])
@pytest.mark.parametrize("layout", ["nhd", "hnd"])
def test_prefill_exact_temperatures(hpc, kpt, temp, layout):
    """Two kv heads, so that HND moves the head stride (with one kv head its bytes equal NHD's)."""
    d = make_prefill_exact_inputs([1024], [1024], 4, 2, 0.3, kpt, kind="peaked",
                                  temperature=temp, layout=layout, seed=3)
    _prefill_case(hpc, f"prefill peaked kpt={kpt} T{temp} {layout}", d, kpt)


@pytest.mark.parametrize("kpt", [False, True])
@pytest.mark.parametrize("climb", [0.70, 0.80, 20.0, -30.0])
@pytest.mark.parametrize("layout", ["nhd", "hnd"])
def test_prefill_exact_lazy_max_schedules(hpc, kpt, climb, layout):
    """Tile maxima climbing 0.70 log2 (no rescale on every tile, P near 430), 0.80 (a rescale
    per tile), 20 (only the last visited tile counts) or falling 30 (P underflows to 0); GQA 4/2."""
    d = make_prefill_exact_inputs([640, 300], [640, 700], 4, 2, 0.3, kpt, kind="sched",
                                  climb=climb, layout=layout, seed=4)
    _prefill_case(hpc, f"prefill sched kpt={kpt} climb{climb} {layout}", d, kpt)


@pytest.mark.parametrize("kpt", [False, True])
def test_prefill_exact_ragged_and_chunked(hpc, kpt):
    q_lens, kv_lens = [1, 130, 257, 64], [1, 130, 900, 1000]
    d = make_prefill_exact_inputs(q_lens, kv_lens, 8, 2, 0.4, kpt, kind="peaked", seed=8)
    _prefill_case(hpc, f"prefill ragged kpt={kpt}", d, kpt)
    d = make_prefill_exact_inputs(q_lens, kv_lens, 8, 2, None, kpt, kind="sched", climb=0.7,
                                  layout="hnd", seed=9)
    _prefill_case(hpc, f"prefill ragged dense kpt={kpt}", d, kpt)


@pytest.mark.parametrize("kpt", [False, True])
def test_prefill_exact_short_mask_and_dead_tile(hpc, kpt):
    d = make_prefill_exact_inputs([1024], [1024], 4, 1, 0.3, kpt, kind="peaked", mask_cols=5,
                                  seed=10)
    _prefill_case(hpc, f"prefill short mask kpt={kpt}", d, kpt)
    d = make_prefill_exact_inputs([512], [512], 4, 1, 0.0, kpt, kind="peaked", seed=12,
                                  dead_tile=(0, 2, 1))
    _prefill_case(hpc, f"prefill dead tile kpt={kpt}", d, kpt)


@pytest.mark.parametrize("kpt", [False, True])
@pytest.mark.parametrize("num_seq_q", [100, 1500])
@pytest.mark.parametrize("layout", ["nhd", "hnd"])
def test_dense_prefill_exact(hpc, kpt, num_seq_q, layout):
    d = make_prefill_exact_inputs([num_seq_q] * 2, [3904] * 2, 4, 1, None, kpt, kind="peaked",
                                  temperature=4.0, layout=layout, seed=num_seq_q)
    _prefill_case(hpc, f"dense prefill kpt={kpt} q{num_seq_q} {layout}", d, kpt, dense_api=True)
