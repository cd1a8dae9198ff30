"""Generate tests/golden/norm_*.npz and masked_act_*.npz from the REFERENCE's own ground-truth
functions, the way tests/golden/make_golden.py does for the other ops (and with its helpers).

Run in the build container only (needs the reference checkout; the GPU box never runs this):
    python tests/golden/make_golden_norm_act.py

`reference_torch_rmsnorm_with_scale` and `reference_torch_rmsnorm` (reference
tests/test_normalization.py:13-28) and `ref_masked_act_mul_and_quant`,
`ref_masked_act_mul_and_blockwise_quant` (reference tests/test_act.py:31-39, 105-115) are
AST-extracted and executed unmodified on CPU tensors, on inputs drawn as the reference tests draw
them (torch.rand weight of shape (1, H), randn x, scale 2.5 or [2.5, 5]; randn gate_up and scale).
"""
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
from make_golden import OUT, REF, _bf16_bits, extract_many, u8  # noqa: E402

NORM = REF / "tests/test_normalization.py"
ACT = REF / "tests/test_act.py"


def norm_case(H, T, is_moe, seed):
    ns = extract_many(NORM, ["reference_torch_rmsnorm_with_scale", "reference_torch_rmsnorm"])
    g = torch.Generator().manual_seed(seed)
    w = torch.rand((1, H), generator=g).to(torch.bfloat16)
    x = torch.randn(T, H, generator=g).to(torch.bfloat16)
    scale = torch.tensor([2.5, 5.0] if is_moe else [2.5], dtype=torch.float32)
    eps = 1e-6
    gt = ns["reference_torch_rmsnorm_with_scale"](x, w, scale[0], eps)
    gt2 = ns["reference_torch_rmsnorm_with_scale"](x, w, scale[-1], eps)
    gt32 = ns["reference_torch_rmsnorm"](x, w, eps)
    tag = f"norm_h{H}_{'moe' if is_moe else 'plain'}"
    np.savez_compressed(OUT / f"{tag}.npz", x=_bf16_bits(x), w=_bf16_bits(w), scale=scale.numpy(),
                        eps=np.array([eps]), gt=_bf16_bits(gt), gt2=_bf16_bits(gt2),
                        gt_fp32=gt32.float().numpy())
    print("wrote", tag, tuple(gt.shape))


def masked_case(tag, counts, T_max, C, seed):
    ns = extract_many(ACT, ["ref_masked_act_mul_and_quant", "ref_masked_act_mul_and_blockwise_quant"])
    g = torch.Generator().manual_seed(seed)
    E = len(counts)
    gate_up = torch.randn((E * T_max, 2 * C), generator=g).to(torch.bfloat16)
    scale = torch.randn((1,), generator=g)
    cnt = torch.tensor(counts, dtype=torch.int32)
    gt = ns["ref_masked_act_mul_and_quant"](gate_up, scale, cnt)
    gtb, gts = ns["ref_masked_act_mul_and_blockwise_quant"](gate_up, cnt)
    np.savez_compressed(OUT / f"masked_act_{tag}.npz", gate_up=_bf16_bits(gate_up), scale=scale.numpy(),
                        num_per_expert=cnt.numpy(), T_max=np.array([T_max]), gt=u8(gt),
                        gt_block=u8(gtb), gt_scale=gts.numpy())
    print("wrote masked_act", tag, tuple(gt.shape))


if __name__ == "__main__":
    for i, H in enumerate((320, 4096, 5120)):
        for is_moe in (False, True):
            norm_case(H, 17 if H < 1024 else 5, is_moe, seed=70 + i)
    masked_case("a", [0, 5, 12, 3], 12, 256, seed=81)
    masked_case("b", [9, 1, 16, 0, 7, 16], 16, 384, seed=82)
