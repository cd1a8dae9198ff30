"""One small invocation of every hot-path op (decode both quant types, prefill both, bf16 prefill
dense and paged, blockwise + per-tensor MoE, bf16 MoE, route GEMM, allreduce with a simulated
peer (P2P high-throughput, Lamport one-shot and two-shot), rope, the Stem mask stages,
fused RMSNorm -> FP8, the masked activation quantisers, the speculative sampler, MLA decode and
prefill, and a multi-row split of the rotated decode walk in the FP8 and MLA decode kernels),
meant to run under compute-sanitizer:

    compute-sanitizer --tool memcheck  python tools/sanitize_smoke.py
    compute-sanitizer --tool synccheck python tools/sanitize_smoke.py
    compute-sanitizer --tool racecheck python tools/sanitize_smoke.py

(the reference's replay harness does the same per call: conftest.py:74-159). Results are checked
against the oracle so that a clean sanitizer run is also a correct one."""
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "hpc-ops_b200"))
import torch  # noqa: E402

import hpc  # noqa: E402
from oracle import attention as oa, moe as om, prefill as op, rope as orp  # noqa: E402
from synth import rope as sr  # noqa: E402


def cuda(d):
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in d.items()}


def main():
    which = set(sys.argv[1:]) or {"decode", "prefill", "prefill_bf16", "moe", "moe_bf16", "gemm",
                                  "allreduce", "rope", "stem", "norm_act", "spec", "mla",
                                  "mla_prefill", "walk"}
    if "decode" in which:
        B, hkv, hq = 3, 2, 8
        lens = [300, 129, 64]
        d = oa.make_decode_fp8_inputs(B, 1, lens, hkv, hq, seed=1, device="cuda")
        tm = hpc.get_attention_decode_task_workspace(B, max(lens), hkv, 64)
        hpc.assign_attention_decode_task(d["kv_lens_total"], tm, hkv, 1, True, 64)
        y = hpc.attention_decode_fp8(d["q"], d["kvcache"][:, 0], d["kvcache"][:, 1], d["block_ids"],
                                     d["kv_lens_total"], d["q_scale"], d["k_scale"], d["v_scale"],
                                     mtp=0, new_kv_included=True, task_map=tm)
        c = {k: v.cpu() for k, v in d.items()}
        gt = oa.decode_fp8_kvpertensor(c["q"], c["kvcache"][:, 0], c["kvcache"][:, 1], c["block_ids"],
                                       c["kv_lens_total"], c["q_scale"], c["k_scale"], c["v_scale"], 1)
        assert torch.allclose(y.float().cpu(), gt.float(), atol=0.2)
        d = oa.make_decode_fp8_kpt_inputs(B, 1, lens, hkv, hq, seed=2, device="cuda")
        y = hpc.attention_decode_fp8(d["q"], d["kcache"], d["vcache"], d["block_ids"], d["kv_lens_total"],
                                     d["q_scale"], d["k_scale"], d["v_scale"], mtp=0, new_kv_included=True,
                                     quant_type=hpc.QuantType.QPERTOKEN_PERHEAD_KPERTOKEN_PERHEAD_VPERHEAD,
                                     task_map=tm)
        c = {k: v.cpu() for k, v in d.items()}
        gt = oa.decode_fp8_kpertoken(c["q"], c["kcache"], c["vcache"], c["block_ids"], c["kv_lens_total"],
                                     c["q_scale"], c["k_scale"], c["v_scale"], 1)
        assert torch.allclose(y.float().cpu(), gt.float(), atol=0.1)
        print("decode ok")
    if "prefill" in which:
        for kpt in (False, True):
            d = op.make_inputs([300], [300], 4, 1, 0.5, kpt, seed=3)
            c = cuda(d)
            qt = (hpc.QuantType.QPERTOKEN_PERHEAD_KPERTOKEN_PERHEAD_VPERHEAD if kpt
                  else hpc.QuantType.QPERTOKEN_PERHEAD_KPERTENSOR_VPERTENSOR)
            y = hpc.attention_with_kvcache_blocksparse_prefill_fp8(
                c["q"], c["kcache"], c["vcache"], c["qscale"], c["kscale"], c["vscale"], c["cu_seqlens_q"],
                c["block_ids"], c["seqlens_kv"], d["max_q"], quant_type=qt,
                block_mask=c["block_mask"].to(torch.uint8).contiguous())
            gt = op.blocksparse_prefill(d["q"], d["kcache"], d["vcache"], d["qscale"], d["kscale"],
                                        d["vscale"], d["cu_seqlens_q"], d["seqlens_kv"], d["block_ids"],
                                        d["block_mask"], kpt)
            assert torch.allclose(y.float().cpu(), gt.float(), atol=0.1)
        print("prefill ok")
    if "prefill_bf16" in which:
        from oracle import prefill_bf16 as ob
        from synth import prefill_bf16 as sb
        for case in (sb.GRID[0], sb.GRID[3]):  # dense; paged with 16-token pages and an sq = 0 slot
            d = sb.make_exact_case(case, "needle", device="cuda")
            if d["op"] == "dense":
                y = hpc.attention_prefill_bf16(d["q"], d["k"], d["v"], d["seqlens_q"],
                                               d["cu_seqlens_q"], d["max_q"])
            else:
                y = hpc.attention_with_kvcache_prefill_bf16(d["q"], d["kcache"], d["vcache"],
                                                            d["cu_seqlens_q"], d["block_ids"],
                                                            d["seqlens_kv"], d["max_q"])
            r = ob.check(y.cpu(), {k: (v.cpu() if isinstance(v, torch.Tensor) else v)
                                   for k, v in d.items()})
            assert r["ok_a"] and r["ok_b"], r
        print("prefill_bf16 ok")
    if "moe" in which:
        d = om.make_moe_blockwise_inputs(96, 4, 256, 256, 8, 1, False, seed=5)
        c = cuda(d)
        y = hpc.fuse_moe_blockwise_fp8(c["x"], c["x_scale"], c["gate_up_weight"], c["gate_up_weight_scale"],
                                       c["down_weight"], c["down_weight_scale"], c["topk_ids"],
                                       c["topk_scale"], 0, 8)
        gt = om.fuse_moe_blockwise(d["x"], d["x_scale"], d["gate_up_weight"], d["gate_up_weight_scale"],
                                   d["down_weight"], d["down_weight_scale"], d["topk_ids"],
                                   d["topk_scale"], 0, None)
        err = (y.float().cpu() - gt.float()).abs()
        assert float((err > 0.01 + 0.01 * gt.float().abs()).float().mean()) < 1e-3
        print("moe ok")
    if "moe_bf16" in which:
        from oracle import moe_bf16 as ob
        from synth.moe_bf16 import make_moe_bf16_inputs
        d = make_moe_bf16_inputs(40, 2, 256, 256, 16, routing="other_rank", size_ep=2, rank_ep=1,
                                 shared=True, seed=6)
        c = cuda(d)
        y = hpc.fuse_moe_bf16(c["x"], c["gate_up_weight"], c["down_weight"], c["topk_ids"],
                              c["topk_scale"], 1, 16, shared_output=c["shared_output"])
        gt = ob.reference_fp32(d["x"], d["gate_up_weight"], d["down_weight"], d["topk_ids"],
                               d["topk_scale"], 1, 16, d["shared_output"])
        torch.testing.assert_close(y.float().cpu(), gt.float(), atol=2e-2, rtol=2e-2)
        print("moe_bf16 ok")
    if "gemm" in which:
        from oracle import gemm as og
        x, w, wh, wl, scale = og.make_inputs(48, 192, 1024, device="cuda")
        ws = hpc.get_gemm_bf16xfp32_workspace(192, 4096)
        y = hpc.gemm_bf16xfp32(x, wh, wl, scale, True, True, ws)
        ref = og.gemm_split_exact(x, wh, wl, scale)
        assert float(((y.double() - ref).abs().max() / ref.abs().max())) < 1e-4
        # split 8 over 4 K steps (k = 200, ragged): CTAs 4..7 of every cluster have no K step
        from oracle import gemm_exact as ge
        x, _, wh, wl, scale = og.make_inputs(129, 192, 200, device="cuda")
        y = torch.empty((129, 192), device="cuda")
        hpc._ffi.check(hpc._ffi.lib.hpc_gemm_bf16xfp32_async(
            hpc._ffi.ptr(y), None, None, hpc._ffi.ptr(x), hpc._ffi.ptr(wh), hpc._ffi.ptr(wl), 129, 192, 200,
            scale, 1, 8, 128, 1, 0, hpc._ffi.stream_of(x)), "gemm_bf16xfp32")
        ye, _, E = ge.route_exact(x.cpu(), wh.cpu(), wl.cpu(), scale, 8)
        ge.route_accumulation_ratio(y.cpu(), ye, E)
        # 1x128 quantiser -> dense blockwise FP8 GEMM, split 8 over 17 K blocks, ragged N = 576
        from oracle import gemm_blockwise as obw
        from synth import gemm_blockwise as sbw
        a = sbw.quant_input(3, 2176, seed=1).cuda()
        q, qs = hpc.blockwise_fp8_quant(a)
        assert obw.quant_mismatch(q.cpu(), qs.cpu(), *obw.quant(a.cpu())) == (0, 0)
        d = sbw.make_inputs(sbw.CASES[4])
        c = cuda(d)
        y = hpc.gemm_blockwise_fp8(c["x"], c["xs"], c["w"], c["ws"])
        split = hpc._ffi.lib.hpc_gemm_blockwise_fp8_config(3, 576, 2176)
        obw.check(y.cpu(), *obw.gemm_exact(d["x"], d["xs"], d["w"], d["ws"], split)[:2])
        # scatter grouped GEMM with indices the gather clamps into the pool (-1, pool_rows)
        from synth import gemm_exact as sg
        d = sg.make_scatter_case(sg.SCATTER_CASES[0])
        c = cuda(d)
        G = d["w"].size(0)
        z = torch.zeros(G + 1, dtype=torch.int32, device="cuda")
        out = torch.ops.hpc.group_gemm_fp8_scatter_cp_async(c["pool"], c["w"], c["y_scale"], c["row_indices"],
                                                            c["seqlens"], c["cu_seqlens"], z[:G], z, False)
        compact = d["pool"][ge.scatter_rows(d["row_indices"], d["pool"].size(0))]
        rows = ge.rows_to_check(d["seqlens"], d["cu_seqlens"], 1, 1)
        ye, B, _ = ge.grouped_pertensor_exact(compact, d["w"], d["seqlens"], d["cu_seqlens"], d["y_scale"], rows)
        ge.check_down(out.cpu()[rows], ye, B)
        print("gemm ok")
    if "allreduce" in which:
        from oracle import allreduce_exact as ox
        from synth import allreduce as sa
        # the P2P transports with a simulated peer on one device: high-throughput (mode 2), then
        # the Lamport kernel one-shot and two-shot, so memcheck sees every peer address
        c = sa.make_case("signature", 2, 6, 264, seed=1)
        args = (c["xs"], c["residual"], c["weight"], c["eps"])
        sim = sa.HtSim(c["xs"], 264)
        res, w = c["residual"].cuda(), c["weight"].cuda()
        ores = torch.empty_like(res)
        for rank in range(2):
            sim.launch(rank, 3 * rank, 3 * rank + 3, res[3 * rank:], w, c["eps"], ores[3 * rank:], 1)
        torch.cuda.synchronize()
        assert ox.check(ores.cpu(), sim.outs[1].cpu(), *args)["ok"]
        for proto in (0, 1):
            c = sa.make_case("lamport", 2, 5, 264, seed=2)
            args = (c["xs"], c["residual"], c["weight"], c["eps"])
            out = torch.empty(5, 264, dtype=torch.bfloat16, device="cuda")
            ores = torch.empty_like(out)
            sa.ll_sim(*args, 1, proto, sa.ll_buf_bytes(5, 2, 264, True), out, ores)
            torch.cuda.synchronize()
            assert ox.check(ores.cpu(), out.cpu(), *args, kernel="ll")["ok"]
        print("allreduce ok")
    if "rope" in which:
        d = sr.make_inputs(3, True, None, 8, 2, 128, seed=7, max_num_kv_blocks=32)
        c = cuda(d)
        q = hpc.rope_norm_store_kv(c["kcache"], c["vcache"], c["qkv"], c["cos_sin"], c["num_seqlen"],
                                   c["q_index"], c["kv_indices"], True, c["q_norm_w"], c["k_norm_w"],
                                   qk_norm_policy=2)
        kc, vc = d["kcache"].clone(), d["vcache"].clone()
        ref = orp.rope_norm_store_kv(kc, vc, d["qkv"], d["cos_sin"], d["num_seqlen"], d["q_index"],
                                     d["kv_indices"], d["q_norm_w"], d["k_norm_w"], 2)
        assert torch.allclose(q.float().cpu(), ref.float(), atol=8e-2) and torch.equal(c["vcache"].cpu(), vc)
        print("rope ok")
    if "stem" in which:
        import numpy as np
        from oracle import stem as ost
        from synth import stem as sst
        for quant, page, layout in ((1, 64, "nhd"), (0, 32, "hnd")):
            d = sst.make_inputs([300, 77, 0], [1100, 3000, 200], 4, 2, page, layout, quant, seed=9)
            c = cuda(d)
            kflat, vbias = hpc.stem_oam_prep_paged_kv(c["kcache"], c["vcache"], c["kscale"], c["vscale"],
                                                      c["kv_indices"], c["kv_seq_lens"], 0.3,
                                                      quant_type=hpc.QuantType(quant))
            qflat = hpc.stem_oam_prep_varlen_q(c["q"], c["qscale"], c["q_seq_lens"], c["cu_seqlens_q"])
            lg = hpc.stem_oam_gemm(qflat, kflat, vbias, c["q_seq_lens"], c["kv_seq_lens"])
            mask = hpc.stem_tpd(lg, c["q_seq_lens"], c["kv_seq_lens"], c["kv_seq_lens"], alpha=0.5)
            kv = ost.kv_prep(d["kcache"], d["vcache"], d["kscale"], d["vscale"], d["kv_indices"],
                             d["kv_seq_lens"], 0.3, quant)
            for b, o in enumerate(kv):
                nkb = o["vbias"].shape[1]
                assert (np.abs(kflat[b, :, :nkb].double().cpu().numpy() - o["kflat"]) <= o["kflat_bound"]).all()
            y, bound, dead = ost.gemm(qflat.cpu(), kflat.cpu(), vbias.cpu(), d["q_seq_lens"], d["kv_seq_lens"])
            lgc = lg.double().cpu().numpy()
            assert np.array_equal(np.isneginf(lgc), dead) and (np.abs(lgc - y)[~dead] <= bound[~dead]).all()
            want = ost.tpd(lg, d["q_seq_lens"], d["kv_seq_lens"], d["kv_seq_lens"], alpha=0.5)
            assert np.array_equal(mask.cpu().numpy(), want)
        wide = sst.adversarial_logits(1, 2, 3, 1500, seed=1)
        ql, kl = torch.tensor([300], dtype=torch.int32), torch.tensor([1500 * 128], dtype=torch.int32)
        m = hpc.stem_tpd(wide.cuda(), ql.cuda(), kl.cuda(), kl.cuda())
        assert np.array_equal(m.cpu().numpy(), ost.tpd(wide, ql, kl, kl))
        print("stem ok")
    if "norm_act" in which:
        from oracle import masked_act as oact, normalization as onorm
        from synth import act as sact, normalization as snorm
        d = snorm.make_inputs(5, 1032, seed=11, device="cuda")
        out = hpc.fused_rmsnorm_with_scale(d["x"], d["w"], d["eps"], d["scale"], True)
        res = onorm.check(out, d["x"], d["w"], d["eps"], d["scale"], True)
        assert not onorm.failed(res), res
        for blockwise in (False, True):
            d = sact.make_inputs(6, 5, 256, seed=12, device="cuda")
            sent = sact.sentinel_outputs(30, 256, device="cuda")
            o, s = sent[0].clone(), sent[1].clone()
            if blockwise:
                hpc.masked_act_mul_and_blockwise_quant(d["gate_up"], d["num_per_expert"], o, s)
            else:
                hpc.masked_act_mul_and_quant(d["gate_up"], d["scale"], d["num_per_expert"], o)
            res = oact.masked_check(o, s if blockwise else None, d["gate_up"], d["num_per_expert"], 5,
                                    sent, scale=d["scale"])
            assert oact.masked_ok(res), res
        print("norm_act ok")
    if "spec" in which:
        import numpy as np
        from oracle import spec_sampler as osp
        from synth import spec_sampler as ssp
        for probs in (False, True):  # given noise, then the kernel's own (checked for range only)
            case = ssp.make_case(13, 6, 2, 4096, torch.bfloat16, probs=probs, pad=128)
            n = case["np"]
            dev = {k: torch.from_numpy(np.ascontiguousarray(n[k])).cuda() if n[k] is not None else None
                   for k in ("draft_token_ids", "draft_probs", "temperature", "uniform", "noise")}
            logits = case["store_t"].cuda()[:, :4096]
            out, nacc = hpc.fused_speculative_sampler(
                logits, dev["draft_token_ids"], draft_probs=dev["draft_probs"], temperature=dev["temperature"],
                uniform=dev["uniform"], gumbel_noise=dev["noise"])
            want, want_n = osp.spec_sample(n["store"], 4096, n["draft_token_ids"], draft_probs=n["draft_probs"],
                                           temperature=n["temperature"], uniform=n["uniform"], noise=n["noise"])
            assert np.array_equal(out.cpu().numpy(), want) and np.array_equal(nacc.cpu().numpy(), want_n)
            out, nacc = hpc.fused_speculative_sampler(logits, dev["draft_token_ids"], draft_probs=dev["draft_probs"],
                                                      temperature=dev["temperature"], seed=3)
            o = out.cpu().numpy()
            assert ((o >= 0) & (o < 4096) | (o == -1)).all()
        print("spec ok")
    if "mla" in which:
        # absorbed MLA decode: two query tiles, a split pair and NaN in the unused cache slots
        from oracle import attention_mla as oml
        from synth import attention_mla as sml
        d = sml.make_case([700, 65], 128, 0, seed=1, num_total_ctas=hpc._ffi.sm_count(),
                          min_process_len=64)
        T = oml.num_tiles(128, 1)
        tm = hpc.get_attention_decode_task_workspace(2, d["block_ids"].size(1) * 64 + 1, T, 64)
        lens = d["lens_total"].cuda()
        hpc.assign_attention_decode_task(lens, tm, T, 1, True, 64)
        y = hpc.attention_decode_mla_bf16(d["q"].cuda(), d["kv"].cuda(), d["block_ids"].cuda(), lens,
                                          d["scale"], mtp=0, new_kv_included=True, task_map=tm)
        r = oml.check(y.float().cpu(), d)
        assert r["ok_a"] and r["ok_b"], r
        print("mla ok")
    if "walk" in which:
        # the rotated bin walk (oracle/decode_walk.py): one multi-row split call for each kernel
        from oracle import attention_mla as oml
        from oracle import decode_walk as dw
        from synth import attention_mla as sml
        from synth.attention_exact import make_decode_exact_inputs
        ctas = hpc._ffi.sm_count()
        for kind, T, sq, h in (("fp8", 2, 1, 8), ("mla", 2, 1, 128)):
            lens = [2000 + 347 * i for i in range(12)]
            walks = dw.walk(dw.task_map(lens, ctas, T, sq, 64), len(lens), T)
            assert dw.path_counts(walks, sq).get("d"), "no multi-row split walk"
            dlens = torch.tensor(lens, dtype=torch.int32, device="cuda")
            tm = hpc.get_attention_decode_task_workspace(len(lens), max(lens) + sq, T, 64)
            hpc.assign_attention_decode_task(dlens, tm, T, sq, True, 64)
            if kind == "fp8":
                d = make_decode_exact_inputs("needle", lens, sq, T, h, seams=dw.seam_keys(walks),
                                             seed=5)
                c = cuda(d)
                y = hpc.attention_decode_fp8(c["q"], c["kvcache"][:, 0], c["kvcache"][:, 1],
                                             c["block_ids"], dlens, c["q_scale"], c["k_scale"],
                                             c["v_scale"], mtp=0, new_kv_included=True,
                                             quant_type=hpc.QuantType.QPERTOKEN_PERHEAD_KPERTENSOR_VPERTENSOR,
                                             splitk=True, task_map=tm)
                from oracle import attention_exact as ox
                k, v = d["kvcache"][:, 0], d["kvcache"][:, 1]
                ex, bnd = ox.decode_fp8_exact(d["q"], k, v, d["block_ids"], d["kv_lens_total"],
                                              d["q_scale"], d["k_scale"], d["v_scale"], sq)
                lossy = oa.decode_fp8_kvpertensor(d["q"], k, v, d["block_ids"], d["kv_lens_total"],
                                                  d["q_scale"], d["k_scale"], d["v_scale"], sq)
                ox.assert_exact(y.cpu(), ex, bnd, lossy, "walk fp8")
            else:
                d = sml.make_case(lens, h, 0, seed=5, kind="needle", num_total_ctas=ctas,
                                  min_process_len=64, seams=dw.seam_keys(walks))
                y = hpc.attention_decode_mla_bf16(d["q"].cuda(), d["kv"].cuda(), d["block_ids"].cuda(),
                                                  dlens, d["scale"], mtp=0, new_kv_included=True,
                                                  task_map=tm)
                r = oml.check(y.float().cpu(), d)
                assert r["ok_a"] and r["ok_b"], r
            torch.cuda.synchronize()
        print("walk ok")
    if "mla_prefill" in which:
        # MLA prefill: two ragged requests, one over a prefix, NaN past the last key
        from oracle import prefill_mla as omp
        from synth import prefill_mla as smp
        d = smp.make_case([130, 70], [300, 70], 4, seed=1, kind="edge")
        y = hpc.attention_prefill_mla_bf16(d["q"].cuda(), d["k_nope"].cuda(), d["k_pe"].cuda(),
                                           d["v"].cuda(), d["cu_seqlens_q"].cuda(),
                                           d["cu_seqlens_kv"].cuda(), d["max_q"], d["scale"])
        r = omp.check(y.float().cpu(), d)
        assert r["ok_a"] and r["ok_b"], r
        print("mla_prefill ok")
    torch.cuda.synchronize()
    print("smoke ok")


if __name__ == "__main__":
    main()
