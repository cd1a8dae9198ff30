"""Stem block-mask stages on the GPU, each against oracle/stem.py from the kernel's own inputs to
that stage, then end to end, under graph capture, and feeding the block-sparse FP8 prefill."""
import numpy as np
import pytest
import torch

from oracle import stem as os_
from synth import stem as ss

pytestmark = pytest.mark.gpu


def _cuda(d):
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in d.items()}


def _run_prep(hpc, c):
    qt = hpc.QuantType(c["quant_type"])
    kflat, vbias = hpc.stem_oam_prep_paged_kv(c["kcache"], c["vcache"], c["kscale"], c["vscale"],
                                              c["kv_indices"], c["kv_seq_lens"], 0.3, quant_type=qt)
    qflat = hpc.stem_oam_prep_varlen_q(c["q"], c["qscale"], c["q_seq_lens"], c["cu_seqlens_q"])
    return kflat, vbias, qflat


def _within(x, y, bound, what):
    err = np.abs(x - y)
    bad = ~(err <= bound)
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.size} outside the bound, worst "
                           f"err {err[bad].max():.4g} at bound {bound[bad][np.argmax(err[bad])]:.4g}")


@pytest.mark.parametrize("case", range(len(ss.CASES)))
def test_stages(hpc, case):
    ql, kl, hq, hkv, page, layout, quant, alpha = ss.CASES[case]
    d = ss.make_inputs(ql, kl, hq, hkv, page, layout, quant, seed=100 + case)
    c = _cuda(d)
    kflat, vbias, qflat = _run_prep(hpc, c)
    torch.cuda.synchronize()
    # prep stages
    kv = os_.kv_prep(d["kcache"], d["vcache"], d["kscale"], d["vscale"], d["kv_indices"],
                     d["kv_seq_lens"], 0.3, quant)
    qo = os_.q_prep(d["q"], d["qscale"], d["q_seq_lens"], d["cu_seqlens_q"])
    kf, vb, qf = kflat.double().cpu().numpy(), vbias.double().cpu().numpy(), qflat.double().cpu().numpy()
    for b in range(len(ql)):
        nkb, nqb = kv[b]["vbias"].shape[1], qo[b]["qflat"].shape[1]
        _within(kf[b, :, :nkb], kv[b]["kflat"], kv[b]["kflat_bound"], f"kflat b{b}")
        _within(vb[b, :, :nkb], kv[b]["vbias"], kv[b]["vbias_bound"], f"vbias b{b}")
        _within(qf[b, :, :nqb], qo[b]["qflat"], qo[b]["qflat_bound"], f"qflat b{b}")
    # GEMM from the kernel's own prep outputs
    logits = hpc.stem_oam_gemm(qflat, kflat, vbias, c["q_seq_lens"], c["kv_seq_lens"])
    y, bound, dead = os_.gemm(qflat.cpu(), kflat.cpu(), vbias.cpu(), d["q_seq_lens"], d["kv_seq_lens"])
    lg = logits.double().cpu().numpy()
    assert np.array_equal(np.isneginf(lg), dead), "-inf pattern differs"
    _within(lg[~dead], y[~dead], bound[~dead], "logits")
    # TPD bit-exact on the kernel's logits
    prompt = d["kv_seq_lens"] + torch.tensor([0] + [64] * (len(ql) - 1), dtype=torch.int32)
    mask = hpc.stem_tpd(logits, c["q_seq_lens"], c["kv_seq_lens"], prompt.cuda(), alpha=alpha)
    want = os_.tpd(logits, d["q_seq_lens"], d["kv_seq_lens"], prompt, alpha=alpha)
    assert np.array_equal(mask.cpu().numpy(), want)
    # end to end: a bit may differ only next to the row's threshold
    e2e = hpc.stem_paged_kv(c["q"], c["kcache"], c["vcache"], c["qscale"], c["kscale"], c["vscale"],
                            c["kv_indices"], c["cu_seqlens_q"], c["kv_seq_lens"], prompt.cuda(),
                            alpha=alpha, quant_type=hpc.QuantType(quant))
    assert torch.equal(e2e, mask), "stem_paged_kv differs from the staged calls"
    _check_e2e(d, kv, qo, mask.cpu().numpy(), prompt, alpha)


def _check_e2e(d, kv, qo, mask, prompt, alpha):
    """Mask against the fp64 pipeline: bits may differ only where the oracle's logit is within the
    combined prep + GEMM bound of the row's threshold value."""
    B = len(kv)
    hkv = kv[0]["vbias"].shape[0] if kv[0]["vbias"].size else d["kcache"].shape[2]
    differ = 0
    for b in range(B):
        ql, kl = int(d["q_seq_lens"][b]), int(d["kv_seq_lens"][b])
        if ql == 0:
            assert not mask[b].any()
            continue
        qf, qfb = qo[b]["qflat"], qo[b]["qflat_bound"]
        kf, kfb = kv[b]["kflat"], kv[b]["kflat_bound"]
        hq = qf.shape[0]
        g = hq // hkv
        nqb, nkb = qf.shape[1], kf.shape[1]
        dead = os_.neg_inf_mask(ql, kl, nqb, nkb)
        for h in range(hq):
            k, kb_, vb, vbb = kf[h // g], kfb[h // g], kv[b]["vbias"][h // g], kv[b]["vbias_bound"][h // g]
            y = qf[h] @ k.T / 64 + vb
            bnd = (np.abs(qf[h]) @ kb_.T + qfb[h] @ np.abs(k).T + qfb[h] @ kb_.T) / 64 + vbb
            mag = np.abs(qf[h]) @ np.abs(k).T / 64
            bnd = bnd + 2048 * 2.0 ** -23 * mag + os_.half_ulp_bf16(np.abs(y) * 1.01 + bnd) * 2
            yb = torch.from_numpy(np.where(dead, -np.inf, y)).to(torch.bfloat16)
            want = os_.tpd(yb[None, None], d["q_seq_lens"][b:b + 1], d["kv_seq_lens"][b:b + 1],
                           prompt[b:b + 1], alpha=alpha)[0, 0]
            got = mask[b, h, :nqb, :nkb]
            for qr in np.nonzero((got != want).any(1))[0]:
                cols = np.nonzero(got[qr] != want[qr])[0]
                # threshold value of the oracle row: the smallest selected-by-score logit
                keys = os_.ordered_keys(yb[qr].view(torch.int16).numpy().astype(np.uint16))
                fin = np.sort(keys[keys != os_.NON_FINITE])[::-1]
                P = os_.cdiv(int(prompt[b]), 128)
                bud = os_.budget(qr + os_.causal_offset(ql, kl), P, alpha)
                tv = y[qr][keys == fin[min(max(bud, 1), len(fin)) - 1]].min()
                near = np.abs(y[qr, cols] - tv) <= 2 * (bnd[qr, cols] + bnd[qr].max())
                assert near.all(), f"b{b} h{h} q{qr}: bits {cols[~near]} differ away from the threshold"
                differ += len(cols)
    print(f"end-to-end bits next to a threshold that differ: {differ}")


def _planted_oracle_masks(d, prompt, alpha, hq, hkv):
    """fp64 pipeline masks of the planted batch, per request [Hq, Qb, Kb] (None for q_len 0)."""
    kv = os_.kv_prep(d["kcache"], d["vcache"], d["kscale"], d["vscale"], d["kv_indices"],
                     d["kv_seq_lens"], 0.3, d["quant_type"])
    qo = os_.q_prep(d["q"], d["qscale"], d["q_seq_lens"], d["cu_seqlens_q"])
    out = []
    for b in range(len(kv)):
        ql, kl = int(d["q_seq_lens"][b]), int(d["kv_seq_lens"][b])
        if ql == 0:
            out.append(None)
            continue
        nqb, nkb = qo[b]["qflat"].shape[1], kv[b]["kflat"].shape[1]
        dead = os_.neg_inf_mask(ql, kl, nqb, nkb)
        y = np.stack([qo[b]["qflat"][h] @ kv[b]["kflat"][h // (hq // hkv)].T / 64
                      + kv[b]["vbias"][h // (hq // hkv)] for h in range(hq)])
        yb = torch.from_numpy(np.where(dead[None], -np.inf, y)).to(torch.bfloat16)
        out.append(os_.tpd(yb[None], d["q_seq_lens"][b:b + 1], d["kv_seq_lens"][b:b + 1],
                           prompt[b:b + 1], alpha=alpha)[0])
    return out


def _planted(quant, page, layout, hq=8, hkv=2):
    p = ss.PLANTED
    d = ss.make_inputs(p["q_lens"], p["kv_lens"], hq, hkv, page, layout, quant, seed=7, planted=True)
    return d, torch.tensor(p["prompt"], dtype=torch.int32)


@pytest.mark.parametrize("quant,page,layout", [(1, 64, "nhd"), (0, 32, "hnd"), (0, 64, "nhd")])
def test_planted_exact(hpc, quant, page, layout):
    """Late chunks of a 200-block prompt: each row keeps ~25-50 of up to 200 visible blocks. The
    kernel's mask equals the fp64 pipeline's, the top-k really drops visible blocks, and every
    planted block wins in every row."""
    d, prompt = _planted(quant, page, layout)
    c = _cuda(d)
    for alpha in (1.0, 0.5):
        mask = hpc.stem_paged_kv(c["q"], c["kcache"], c["vcache"], c["qscale"], c["kscale"],
                                 c["vscale"], c["kv_indices"], c["cu_seqlens_q"], c["kv_seq_lens"],
                                 prompt.cuda(), alpha=alpha, quant_type=hpc.QuantType(quant)).cpu()
        want = _planted_oracle_masks(d, prompt, alpha, 8, 2)
        dropped = 0
        for b, w in enumerate(want):
            if w is None:
                assert not mask[b].any()
                continue
            ql, kl = int(d["q_seq_lens"][b]), int(d["kv_seq_lens"][b])
            nqb, nkb = w.shape[1], w.shape[2]
            assert np.array_equal(mask[b, :, :nqb, :nkb].numpy(), w), f"b{b} alpha {alpha}"
            visible = ~os_.neg_inf_mask(ql, kl, nqb, nkb)
            dropped += int((visible[None] & (w == 0)).sum())
            assert (w.sum(-1) < visible.sum(-1)[None]).all(), "a row kept every visible block"
            for h in range(8):
                for kb in d["plants"][b][h // 4]:
                    assert mask[b, h, :nqb, kb].all(), f"planted block {kb} missed (b{b} h{h})"
        assert dropped > 0
        print(f"alpha {alpha}: visible blocks dropped by the top-k: {dropped}")


@pytest.mark.parametrize("quant", [1, 0])
def test_planted_mask_prefill_matches_dense(hpc, quant):
    """Where the fp64 softmax mass outside the Stem mask is below 1e-4 for a row, the block-sparse
    prefill with that mask is within 2 * mass * max|v| of the exact dense output, plus the dense
    prefill's exact-check bound."""
    from oracle import attention_exact as ae

    d, prompt = _planted(quant, 64, "nhd")
    c = _cuda(d)
    qt = hpc.QuantType(quant)
    mask = hpc.stem_paged_kv(c["q"], c["kcache"], c["vcache"], c["qscale"], c["kscale"], c["vscale"],
                             c["kv_indices"], c["cu_seqlens_q"], c["kv_seq_lens"], prompt.cuda(),
                             alpha=0.5, quant_type=qt)
    kc, vc = c["kcache"].clone(), c["vcache"].clone()  # the prefill reads whole pages: clear poison
    kc.view(torch.uint8)[kc.view(torch.uint8) == ss.NAN_E4M3] = 0
    vc.view(torch.uint8)[vc.view(torch.uint8) == ss.NAN_E4M3] = 0
    y = hpc.attention_with_kvcache_blocksparse_prefill_fp8(
        c["q"], kc, vc, c["qscale"], c["kscale"], c["vscale"], c["cu_seqlens_q"], c["kv_indices"],
        c["kv_seq_lens"], int(d["q_seq_lens"].max()), qt, block_mask=mask).double().cpu()
    kcc, vcc, m = kc.cpu(), vc.cpu(), mask.cpu()
    exact, bound = ae.prefill_fp8_exact(d["q"], kcc, vcc, d["qscale"], d["kscale"], d["vscale"],
                                        d["cu_seqlens_q"], d["kv_seq_lens"], d["kv_indices"], None,
                                        k_per_token=quant == 0)
    hq, g, checked = 8, 4, 0
    for b in range(2):
        s0, s1 = int(d["cu_seqlens_q"][b]), int(d["cu_seqlens_q"][b + 1])
        nq, nkv = s1 - s0, int(d["kv_seq_lens"][b])
        vis = ae.prefill_visible(nq, nkv)[0]
        sel = ae.prefill_visible(nq, nkv, m[b])
        ids = d["kv_indices"][b, :nkv // 64].long()
        for h in range(hq):
            kk = kcc[ids].reshape(-1, 2, 128)[:nkv, h // g].double()
            vv = vcc[ids].reshape(-1, 2, 128)[:nkv, h // g].double()
            ks = (d["kscale"][0] if quant == 1 else 0.75)
            vs = float(d["vscale"][0] if quant == 1 else d["vscale"][h // g])
            s = (d["q"][s0:s1, h].double() @ kk.T) * d["qscale"][b, h, :nq].double()[:, None] * ks
            s = (s / np.sqrt(128)).masked_fill(~vis, -np.inf)
            p_ = torch.softmax(s, -1)
            mass = (p_ * (vis & ~sel[h]).double()).sum(-1)
            ok = mass < 1e-4
            lim = bound[s0:s1, h] + (2 * mass * vv.abs().max() * abs(vs))[:, None]
            err = (y[s0:s1, h] - exact[s0:s1, h]).abs()
            assert (err[ok] <= lim[ok]).all(), f"b{b} h{h}: {float((err - lim)[ok].max()):.3g} over"
            checked += int(ok.sum())
    assert checked > 0.9 * 812 * hq, f"only {checked} rows had mass below 1e-4"


@pytest.mark.parametrize("max_kb", [37, 1024, 1500, 4096])
def test_tpd_adversarial(hpc, max_kb):
    B, H, qb = 2, 3, 9
    x = ss.adversarial_logits(B, H, qb, max_kb, seed=max_kb)
    ql = torch.tensor([qb * 128 - 5, 300], dtype=torch.int32)
    kl = torch.tensor([max_kb * 128 - 77, min(max_kb, 40) * 128], dtype=torch.int32)
    prompt = torch.tensor([max_kb * 128 + 999, 7200 * 2], dtype=torch.int32)
    for alpha in (1.0, 0.5):
        m = hpc.stem_tpd(x.cuda(), ql.cuda(), kl.cuda(), prompt.cuda(), alpha=alpha)
        want = os_.tpd(x, ql, kl, prompt, alpha=alpha)
        assert np.array_equal(m.cpu().numpy(), want), f"alpha {alpha}"


def test_tpd_budget_fma(hpc):
    """Rows whose decay budget depends on the single rounding of the fused multiply-add."""
    cases = []
    for P in range(56, 400):
        for q_pos in range(P):
            if os_.budget(q_pos, P, 0.3) != os_.budget(q_pos, P, 0.3, fma=False):
                cases.append((P, q_pos))
    assert cases, "no budget depends on the fma in this range"
    P, q_pos = cases[0]
    kv = P * 128
    q_len = 128 * (q_pos + 1)
    x = torch.randn(1, 1, q_pos + 1, P).to(torch.bfloat16)
    args = [torch.tensor([v], dtype=torch.int32) for v in (q_len, kv, kv)]
    m = hpc.stem_tpd(x.cuda(), *[a.cuda() for a in args], alpha=0.3)
    assert np.array_equal(m.cpu().numpy(), os_.tpd(x, *args, alpha=0.3))


def test_fp8_kscale_view_and_determinism(hpc):
    d = ss.make_inputs([300, 129], [5000, 700], 8, 2, 64, "nhd", 0, seed=3)
    c = _cuda(d)
    a = _run_prep(hpc, c)
    c8 = dict(c, kscale=c["kscale"].view(torch.float8_e4m3fn))
    b = _run_prep(hpc, c8)
    r = _run_prep(hpc, c)
    # blocks past a request's own length are not written: compare each request's own blocks
    for i, (kl, ql) in enumerate(zip(d["kv_seq_lens"].tolist(), d["q_seq_lens"].tolist())):
        nkb, nqb = os_.cdiv(kl, 128), os_.cdiv(ql, 128)
        for x, y, z, n in zip(a, b, r, (nkb, nkb, nqb)):
            assert torch.equal(x[i, :, :n].view(torch.int16 if x.dtype == torch.bfloat16 else torch.int32),
                               y[i, :, :n].view(torch.int16 if x.dtype == torch.bfloat16 else torch.int32))
            assert torch.equal(x[i, :, :n], z[i, :, :n])


def test_graph_capture_replay(hpc):
    d1 = ss.make_inputs([500, 200], [3000, 800], 8, 2, 64, "nhd", 1, seed=11)
    d2 = ss.make_inputs([500, 200], [3000, 800], 8, 2, 64, "nhd", 1, seed=12)
    c1, c2 = _cuda(d1), _cuda(d2)
    kf, vb, qf = _run_prep(hpc, c1)
    kf2, vb2, qf2 = _run_prep(hpc, c2)
    prompt = c1["kv_seq_lens"].clone()
    ql, kl = c1["q_seq_lens"].clone(), c1["kv_seq_lens"].clone()
    bufs = [qf.clone(), kf.clone(), vb.clone()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):  # warm up outside the capture
        hpc.stem_tpd(hpc.stem_oam_gemm(*bufs, ql, kl), ql, kl, prompt)
    torch.cuda.current_stream().wait_stream(s)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        lg = hpc.stem_oam_gemm(*bufs, ql, kl)
        mk = hpc.stem_tpd(lg, ql, kl, prompt)
    for src in ((qf2, kf2, vb2), (qf, kf, vb)):
        for dst, x in zip(bufs, src):
            dst.copy_(x)
        gr.replay()
        torch.cuda.synchronize()
        lg_e = hpc.stem_oam_gemm(*src, ql, kl)
        mk_e = hpc.stem_tpd(lg_e, ql, kl, prompt)
        assert torch.equal(lg.view(torch.int16), lg_e.view(torch.int16))
        assert torch.equal(mk, mk_e)


@pytest.mark.parametrize("quant", [1, 0])
def test_mask_feeds_blocksparse_prefill(hpc, quant):
    from oracle import attention_exact as ae, prefill as op

    d = ss.make_inputs([300, 260], [2900, 1500], 8, 2, 64, "nhd", quant, seed=21 + quant)
    c = _cuda(d)
    qt = hpc.QuantType(quant)
    mask = hpc.stem_paged_kv(c["q"], c["kcache"], c["vcache"], c["qscale"], c["kscale"], c["vscale"],
                             c["kv_indices"], c["cu_seqlens_q"], c["kv_seq_lens"], c["kv_seq_lens"],
                             alpha=0.5, quant_type=qt)
    # the prefill reads the cache pages it is given: clear the NaN poison of unused rows first
    kc, vc = c["kcache"].clone(), c["vcache"].clone()
    kc.view(torch.uint8)[kc.view(torch.uint8) == ss.NAN_E4M3] = 0
    vc.view(torch.uint8)[vc.view(torch.uint8) == ss.NAN_E4M3] = 0
    y = hpc.attention_with_kvcache_blocksparse_prefill_fp8(
        c["q"], kc, vc, c["qscale"], c["kscale"], c["vscale"], c["cu_seqlens_q"], c["kv_indices"],
        c["kv_seq_lens"], int(d["q_seq_lens"].max()), qt, block_mask=mask)
    cpu = {k: v.cpu() for k, v in dict(q=c["q"], kc=kc, vc=vc).items()}
    exact, bound = ae.prefill_fp8_exact(cpu["q"], cpu["kc"], cpu["vc"], d["qscale"], d["kscale"],
                                        d["vscale"], d["cu_seqlens_q"], d["kv_seq_lens"],
                                        d["kv_indices"], mask.cpu(), k_per_token=quant == 0)
    lossy = op.blocksparse_prefill(cpu["q"], cpu["kc"], cpu["vc"], d["qscale"], d["kscale"],
                                   d["vscale"], d["cu_seqlens_q"], d["kv_seq_lens"], d["kv_indices"],
                                   mask.cpu(), quant == 0)
    ae.assert_exact(y.cpu(), exact, bound, lossy, f"stem mask q{quant}")
