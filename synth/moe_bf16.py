"""Seeded inputs for the bf16 FusedMoE (hpc.fuse_moe_bf16), CPU tensors with O(1) outputs.

x ~ N(0, 1); gate/up weights ~ N(0, 4 / H), so g and u have rms ~2 (where SiLU is far from
linear); down weights ~ N(0, 1 / I) / 1.5, so each expert's output has rms ~1. Weights are drawn one
expert at a time, so the fp32 staging stays at one expert's size at the Mixtral shape.

routing:
  uniform     top-k without repeats over all experts;
  hot         uniform, then slot 0 of ~60 % of tokens goes to one local expert;
  sparse      uniform, for decode batches (num_tokens <= 16): most experts are empty;
  other_rank  ids drawn with repeats over all ranks' experts (use size_ep > 1): some tokens have no
              local expert.
"""
import torch

ROUTINGS = ("uniform", "hot", "sparse", "other_rank")


def make_moe_bf16_inputs(num_tokens, num_topk, hidden, inter, num_expert_total, routing="uniform",
                         size_ep=1, rank_ep=0, shared=False, seed=41):
    g = torch.Generator().manual_seed(seed)
    E = num_expert_total // size_ep
    if routing in ("uniform", "hot", "sparse"):
        assert routing != "sparse" or num_tokens <= 16, "sparse routing is for num_tokens <= 16"
        ids = torch.multinomial(torch.ones((max(num_tokens, 1), num_expert_total)), num_topk,
                                replacement=False, generator=g)[:num_tokens]
        if routing == "hot":
            hot = torch.rand((num_tokens,), generator=g) < 0.6
            ids[hot, 0] = rank_ep * E + min(3, E - 1)
    elif routing == "other_rank":
        ids = torch.randint(0, num_expert_total, (num_tokens, num_topk), generator=g)
    else:
        raise ValueError(f"unknown routing {routing!r}")
    topk_scale = torch.rand((num_tokens, num_topk), generator=g) + 0.1
    topk_scale = topk_scale / topk_scale.sum(dim=1, keepdim=True)
    x = torch.randn((num_tokens, hidden), generator=g).to(torch.bfloat16)
    gu_std = 2.0 / hidden ** 0.5
    d_std = 1.0 / (1.5 * inter ** 0.5)
    guw = torch.empty((E, 2 * inter, hidden), dtype=torch.bfloat16)
    dw = torch.empty((E, hidden, inter), dtype=torch.bfloat16)
    for e in range(E):
        guw[e] = torch.randn((2 * inter, hidden), generator=g) * gu_std
        dw[e] = torch.randn((hidden, inter), generator=g) * d_std
    sh = torch.randn((num_tokens, hidden), generator=g).to(torch.bfloat16) if shared else None
    return dict(x=x, gate_up_weight=guw, down_weight=dw, topk_ids=ids.to(torch.int32).contiguous(),
                topk_scale=topk_scale.float().contiguous(), shared_output=sh, rank_ep=rank_ep,
                num_expert_total=num_expert_total)


def make_group_gemm_bf16_inputs(seqlens, n, k, seed=43):
    """x [sum(seqlens) + 5, k] (5 rows outside every group), w [G, n, k], seqlens, cu_seqlens."""
    g = torch.Generator().manual_seed(seed)
    sl = torch.tensor(seqlens, dtype=torch.int32)
    cu = torch.zeros(len(seqlens) + 1, dtype=torch.int32)
    cu[1:] = torch.cumsum(sl, 0)
    m = int(cu[-1]) + 5
    x = torch.randn((m, k), generator=g).to(torch.bfloat16)
    w = (torch.randn((len(seqlens), n, k), generator=g) / k ** 0.5).to(torch.bfloat16)
    return dict(x=x, weight=w, seqlens=sl, cu_seqlens=cu)
