"""Seeded inputs for the masked per-expert activation quantisers (hpc.masked_act_mul_and_quant,
hpc.masked_act_mul_and_blockwise_quant) that a wrong kernel cannot pass by accident.

* Counts cycle through 0, 1, T_max, T_max + 5 (clamped to T_max), -3 (no rows) and a random
  count, so that every validity rule is exercised and neighbouring experts differ.
* In the first valid row of each expert, 128-column block 0 is all zero (gate 0: sc = 0), and in
  its last valid row block 0 has |silu(g) * u| near 1e-6, where the +1e-8 of 1 / (sc + 1e-8)
  visibly changes the codes. Every other block's largest element lands on +-448 (code 0x7E / 0xFE).
* The output buffers are pre-filled with sentinels (0x5A bytes, a NaN scale pattern) that must
  survive on every invalid row.
"""
import torch

SENTINEL_U8 = 0x5A
SENTINEL_SCALE_BITS = 0x7FA5A5A5  # a NaN whose payload a kernel would not produce


def counts(E, T_max, seed=0):
    g = torch.Generator().manual_seed(seed + 17)
    if E == 1:
        return torch.tensor([int(torch.randint(1, T_max + 1, (1,), generator=g))], dtype=torch.int32)
    pat = [0, 1, T_max, T_max + 5, -3]
    c = [pat[e % 5] if e % 6 != 5 else int(torch.randint(0, T_max + 1, (1,), generator=g))
         for e in range(E)]
    return torch.tensor(c, dtype=torch.int32)


def valid_rows(cnt, T_max):
    """Boolean [E * T_max] of the rows a kernel may read and write."""
    c = cnt.clamp(0, T_max).to(torch.int64)
    t = torch.arange(T_max)
    return (t[None, :] < c[:, None]).reshape(-1)


def make_inputs(E, T_max, C, seed=0, device="cpu"):
    g = torch.Generator().manual_seed(seed * 7919 + E * 101 + T_max * 13 + C)
    N = E * T_max
    x = torch.randn(N, 2 * C, generator=g)
    cnt = counts(E, T_max, seed)
    c = cnt.clamp(0, T_max)
    if C % 128 == 0:
        for e in range(E):
            n = int(c[e])
            if n >= 1:
                x[e * T_max, :128] = 0  # gate 0 -> the whole block 0 is 0
            if n >= 2:
                r = e * T_max + n - 1
                x[r, :128] *= 1e-3
                x[r, C:C + 128] *= 1e-3
    scale = torch.tensor([1.7], dtype=torch.float32)
    return {"gate_up": x.to(torch.bfloat16).to(device), "num_per_expert": cnt.to(device),
            "scale": scale.to(device), "T_max": T_max}


def sentinel_outputs(N, C, device="cpu"):
    out = torch.full((N, C), SENTINEL_U8, dtype=torch.uint8, device=device).view(torch.float8_e4m3fn)
    sc = torch.full((N, C // 128), SENTINEL_SCALE_BITS, dtype=torch.int32, device=device).view(torch.float32)
    return out, sc
