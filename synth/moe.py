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


def _normal_e4m3(shape, g, lo=-4.0, hi=4.0):
    """sign * 2^U(lo, hi) in e4m3: every value is normal (|v| >= 2^-6), mantissas are uniform."""
    mag = torch.exp2(torch.empty(shape).uniform_(lo, hi, generator=g))
    return torch.where(torch.rand(shape, generator=g) < 0.5, -mag, mag).to(torch.float8_e4m3fn)


def _signed_scale(shape, g):
    """Signed O(1) scales: sign * U(0.5, 1.5)."""
    return (torch.rand(shape, generator=g) + 0.5) * (torch.randint(0, 2, shape, generator=g) * 2 - 1)


# E[v^2] of _normal_e4m3 before rounding: E[4^U], U ~ U(-4, 4)
_E4M3_MS = (4.0 ** 4 - 4.0 ** -4) / (8 * 1.3862943611198906)


def make_moe_blockwise_routed_inputs(num_tokens, num_topk, hidden, inter, num_expert_total,
                                     routing="uniform", size_ep=1, rank_ep=0, shared=False,
                                     seed=41):
    """Blockwise FusedMoE inputs (CPU tensors) with O(1) outputs and a choice of routing.

    x and both weights are normal e4m3 values (sign * 2^U(-4, 4)), so every code carries its full
    3-bit mantissa. Activation and weight scales are signed, of size O(1) times a normalisation:
    the Gate-Up scale makes gate and up O(1) (rms ~2, where SiLU is far from linear), and the Down
    scale makes each expert's output O(1). Weight-scale rows are padded to a multiple of 4 with
    random values, so a kernel that read a pad entry would be wrong by O(1).

    routing:
      uniform      top-k without repeats over all experts;
      hot          uniform, then slot 0 of ~60 % of tokens goes to one local expert (repeats allowed);
      sparse       uniform, for decode batches (num_tokens <= 16): most experts are empty;
      other_ranks  ids drawn with repeats over all ranks' experts (use size_ep > 1).
    """
    g = torch.Generator().manual_seed(seed)
    E = num_expert_total // size_ep
    if routing in ("uniform", "hot", "sparse"):
        assert routing != "sparse" or num_tokens <= 16, "sparse routing is for num_tokens <= 16"
        ids = torch.multinomial(torch.ones((num_tokens, num_expert_total)), num_topk,
                                replacement=False, generator=g)
        if routing == "hot":
            hot = torch.rand((num_tokens,), generator=g) < 0.6
            ids[hot, 0] = rank_ep * E + min(3, E - 1)
    elif routing == "other_ranks":
        ids = torch.randint(0, num_expert_total, (num_tokens, num_topk), generator=g)
    else:
        raise ValueError(f"unknown routing {routing!r}")
    topk_scale = torch.rand((num_tokens, num_topk), generator=g) + 0.1
    topk_scale = topk_scale / topk_scale.sum(dim=1, keepdim=True)
    x = _normal_e4m3((num_tokens, hidden), g)
    x_scale = _signed_scale((num_tokens, hidden // 128), g)
    # one expert at a time: the fp32 staging stays at one expert's size at the C3 shape
    guw = torch.stack([_normal_e4m3((2 * inter, hidden), g) for _ in range(E)])
    dw = torch.stack([_normal_e4m3((hidden, inter), g) for _ in range(E)])
    # gate/up rms ~ sqrt(hidden * E[x^2] E[w^2] E[xs^2] E[ws^2]) ~ 2 (E[s^2] of U(0.5, 1.5) ~ 1.08)
    gu_norm = 2.0 / (_E4M3_MS * (hidden * 1.08) ** 0.5)
    guws = _signed_scale((E, 2 * inter // 128, (hidden // 128 + 3) // 4 * 4), g) * gu_norm
    # down_input codes * (amax / 448) ~ silu(g) * u with rms ~1.5; the Down output rms ~ 2
    d_norm = 2.0 / (1.5 * (_E4M3_MS * inter * 1.08) ** 0.5)
    dws = _signed_scale((E, hidden // 128, (inter // 128 + 3) // 4 * 4), g) * d_norm
    sh = torch.randn((num_tokens, hidden), generator=g).to(torch.bfloat16) if shared else None
    return dict(x=x, x_scale=x_scale.float(), gate_up_weight=guw, gate_up_weight_scale=guws.float(),
                down_weight=dw, down_weight_scale=dws.float(), topk_ids=ids.to(torch.int32),
                topk_scale=topk_scale.float(), shared_output=sh, rank_ep=rank_ep,
                num_expert_total=num_expert_total)


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
