"""Synthetic inputs for the blockwise FusedMoE (distributions of reference
tests/test_fuse_moe_blockwise.py:285-319)."""
import torch


def make_moe_blockwise_inputs(num_tokens, num_topk, hidden, inter, num_expert_total, size_ep=1,
                              shared=False, seed=41, device="cpu", wscale_abs=False):
    dev = torch.device(device)
    g = torch.Generator(device=dev).manual_seed(seed)
    E = num_expert_total // size_ep
    topk_ids = torch.multinomial(torch.ones((num_tokens, num_expert_total), device=dev), num_topk,
                                 replacement=False, generator=g).to(torch.int32)
    topk_ids, _ = torch.sort(topk_ids, dim=1)
    topk_scale = torch.rand((num_tokens, num_topk), generator=g, device=dev)
    topk_scale = topk_scale / topk_scale.sum(dim=1, keepdim=True)
    x = (torch.randn((num_tokens, hidden), generator=g, device=dev) / 100).to(torch.float8_e4m3fn)
    x_scale = torch.randn((num_tokens, hidden // 128), generator=g, device=dev)

    def weights(rows, cols):
        w = torch.empty((E, rows, cols), dtype=torch.float8_e4m3fn, device=dev)
        for e in range(E):
            w[e] = torch.randn((rows, cols), generator=g, device=dev).to(torch.float8_e4m3fn)
        return w

    guw = weights(inter * 2, hidden)
    guws = torch.randn((E, inter * 2 // 128, (hidden // 128 + 3) // 4 * 4), generator=g, device=dev)
    dw = weights(hidden, inter)
    dws = torch.randn((E, hidden // 128, (inter // 128 + 3) // 4 * 4), generator=g, device=dev)
    sh = torch.randn((num_tokens, hidden), generator=g, device=dev).to(torch.bfloat16) if shared else None
    return dict(x=x, x_scale=x_scale, gate_up_weight=guw, gate_up_weight_scale=guws, down_weight=dw,
                down_weight_scale=dws, topk_ids=topk_ids, topk_scale=topk_scale, shared_output=sh)


def make_moe_pertensor_inputs(num_tokens, num_topk, hidden, inter, num_expert_total, size_ep=1,
                              rank_ep=0, shared=False, routing="uniform", seed=41):
    """Per-tensor FusedMoE inputs with O(1) outputs: the Gate-Up and Down scales are 1/sqrt(K)
    (times a per-expert factor in [0.5, 1.5]) so that both GEMM outputs are O(1), and the
    activation scale (8) puts the re-quantised Gate-Up activation in e4m3's normal range
    (|codes| ~ 0.5 ... 200); the Down scale divides it out again.
    routing: "uniform" (top-k without repeats over all experts), or "repeat": every token picks
    from 3 small experts of this rank and 2 of another rank, with repeats inside a row, so that
    most local experts are empty and the rest get few rows."""
    g = torch.Generator().manual_seed(seed)
    E = num_expert_total // size_ep
    if routing == "uniform":
        ids = torch.multinomial(torch.ones((num_tokens, num_expert_total)), num_topk,
                                replacement=False, generator=g)
        ids, _ = torch.sort(ids, dim=1)
    else:
        pool = torch.tensor([rank_ep * E + 1, rank_ep * E + E // 2, rank_ep * E + E - 1,
                             ((rank_ep + 1) % size_ep) * E, ((rank_ep + 1) % size_ep) * E + 3])
        ids = pool[torch.randint(0, len(pool), (num_tokens, num_topk), generator=g)]
    topk_scale = torch.rand((num_tokens, num_topk), generator=g) + 0.1
    topk_scale = topk_scale / topk_scale.sum(dim=1, keepdim=True)
    x = torch.randn((num_tokens, hidden), generator=g).to(torch.float8_e4m3fn)
    guw = torch.randn((E, 2 * inter, hidden), generator=g).to(torch.float8_e4m3fn)
    dw = torch.randn((E, hidden, inter), generator=g).to(torch.float8_e4m3fn)
    act_scale = torch.tensor([8.0])
    gus = (torch.rand((E,), generator=g) + 0.5) / hidden ** 0.5
    ds = (torch.rand((E,), generator=g) + 0.5) / inter ** 0.5 / act_scale
    sh = torch.randn((num_tokens, hidden), generator=g).to(torch.bfloat16) if shared else None
    return dict(x=x, gate_up_weight=guw, down_weight=dw, gate_up_scale=gus.float(),
                down_scale=ds.float(), act_scale=act_scale, topk_ids=ids.to(torch.int32),
                topk_scale=topk_scale.float(), shared_output=sh, rank_ep=rank_ep,
                num_expert_total=num_expert_total)
