"""Seeded inputs for hpc.fused_rmsnorm_with_scale that a wrong kernel cannot pass by accident.

* Row RMS drawn log-uniformly from 1e-3 .. 1e2 per row, so that a row normalised with a
  neighbour's r is off by orders of magnitude.
* Row 1 all zero (y = 0 whatever r is) and row 2 with an RMS of 1e-3, where eps = 1e-6 changes
  r by about 30 %: a kernel that adds eps anywhere else fails there.
* A signed weight whose magnitude spans 0.05 .. 4. Columns 0 and 1 (x = 8 before the row RMS is
  applied, w = +-4) are large in every row.
* scale[0] = 1/64 puts the largest outputs past 448 (saturation) and the smallest into e4m3
  subnormals; scale[1] = 0.75 keeps the second copy mostly in range.
"""
import torch

EPS = 1e-6
SCALES = (1.0 / 64, 0.75)


def make_inputs(T, H, seed=0, device="cpu"):
    g = torch.Generator().manual_seed(seed * 1000003 + T * 131 + H)
    rms = 10.0 ** (torch.rand(T, 1, generator=g) * 5 - 3)
    x = torch.randn(T, H, generator=g)
    x[:, :2] = 8.0  # with w[:2] = +-4 below: outputs past 448 * scale[0] of both signs
    x = x * rms
    if T >= 2:
        x[1] = 0
    if T >= 3:
        x[2] = torch.randn(H, generator=g) * 1e-3
    w = (10.0 ** (torch.rand(H, generator=g) * 1.9 - 1.3)) * torch.where(
        torch.rand(H, generator=g) < 0.5, -1.0, 1.0)
    w[0], w[1] = 4.0, -4.0
    scale = torch.tensor(SCALES, dtype=torch.float32)
    return {"x": x.to(torch.bfloat16).to(device), "w": w.to(torch.bfloat16).to(device),
            "scale": scale.to(device), "eps": EPS}
