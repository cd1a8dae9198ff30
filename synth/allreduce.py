"""Inputs for the fused AllReduce + residual + RMSNorm (csrc/allreduce.cu) and the one-GPU drivers
that run its transports with simulated peers.

Families (`make_case`):
  random     randn ranks, residual and gamma (the multi-GPU tests' data); graded under the
             ambiguity rule of oracle.allreduce_exact.
  exact      magnitudes in [2^-6, 2^6) or zero: every fp32 partial sum over up to 16 ranks is
             exact, so s and r are order-independent and must be bit-exact on every transport.
  signature  rank r contributes +-2^r (signs varying by row and column), residual 0 (W <= 8): each
             out_residual value spells out which ranks reached it; a dropped or doubled rank, a
             wrong peer pointer or a slice off by one row gives a wrong bit pattern.
  cancel     x_1 = -x_0 plus a small term, x_0 up to 2^10, further ranks down to 2^-12: a bf16 or
             reordered accumulation beyond the fp32 bound fails.
  eps        rows with mean square 1e-8 ... 1e-4 (eps matters) and all-zero rows.
  lamport    (+0.0, -0.0) pairs, the Lamport sentinel word 0x80000000, in the inputs (scrubbed
             by the kernel before it stores them); for W >= 2 also positions whose exact sum is
             (0, -0) in sign pattern: -0.0 high halves from every rank, low halves +tiny, -tiny
             and +0.0. Their rank-order fp32 sum is (+0, +0), NOT the sentinel: the owner's
             accumulator starts at +0.0 and +0 + -0 = +0, on every transport (multicast only
             broadcasts the owner's sum). So the scrub of the owner's sum (allreduce.cu, two-shot
             owner) cannot be reached from any input, and no test here shows that it matters.
Magnitudes keep H max^2 inside the fp32 range and every nonzero square above its normal range.

Simulated peers (`HtSim`, `ll_sim`): W ranks' buffers on ONE device, launched one rank at a
time. Before each launch every word the kernel can wait on is filled so that the wait is already
satisfied: signal-pad epochs set to 2^30 (the kernel compares modulo 2^32), Lamport slots holding
the peers' rows and a finite poison value elsewhere. No launch depends on the spin limit.
"""
import ctypes

import numpy as np
import torch

from oracle import allreduce_exact as ox

FAMILIES = ("random", "exact", "signature", "cancel", "eps", "lamport")
# every bucket of both dispatch tables, plus widths that leave lanes idle (264, 2056, 8200, 16392)
HIDDENS = (8, 256, 264, 512, 1024, 2048, 2056, 4096, 7168, 8192, 8200, 16384, 16392, 32768)
TOKENS = (1, 2, 7, 129, 4096)
EPS = (1e-6, 1e-5)
SENTINEL = -2147483648  # int32 view of 0x80000000
POISON = 0x5A5A5A5A     # finite bf16 pair (1.54e16): a wrong read fails the value check
ARRIVED = 1 << 30       # signal-pad epoch every simulated peer has "already posted"


def _grid(g, shape, emin, emax, pzero=0.0):
    """Random bf16 values sign * (1 + k/128) * 2^e, e in [emin, emax], zero with probability pzero."""
    e = torch.randint(emin, emax + 1, shape, generator=g).double()
    k = torch.randint(0, 128, shape, generator=g).double()
    s = torch.randint(0, 2, shape, generator=g).double() * 2 - 1
    v = s * (1 + k / 128) * torch.pow(2.0, e)
    if pzero:
        v[torch.rand(shape, generator=g) < pzero] = 0
    return v.to(torch.bfloat16)


def make_case(family, W, T, H, seed=0, eps=1e-6):
    """dict(xs=[W x [T, H] bf16], residual [T, H] bf16, weight [H] bf16, eps)."""
    g = torch.Generator().manual_seed(seed * 7919 + W * 131 + T * 17 + H)
    weight = _grid(g, (H,), -2, 1)
    shape = (T, H)
    if family == "random":
        xs = [torch.randn(shape, generator=g).to(torch.bfloat16) for _ in range(W)]
        residual = torch.randn(shape, generator=g).to(torch.bfloat16)
        weight = torch.randn((H,), generator=g).to(torch.bfloat16)
    elif family == "exact":
        xs = [_grid(g, shape, -6, 5, 0.1) for _ in range(W)]
        residual = _grid(g, shape, -6, 5, 0.1)
    elif family == "signature":
        assert W <= 8, "signature values need W <= 8 significant bits"
        xs = [((torch.randint(0, 2, shape, generator=g) * 2 - 1) * 2.0 ** r).to(torch.bfloat16)
              for r in range(W)]
        residual = torch.zeros(shape, dtype=torch.bfloat16)
    elif family == "cancel":
        x0 = _grid(g, shape, 0, 10)
        xs = [x0]
        if W > 1:
            xs.append(ox.to_bf16(-ox.f64(x0) + ox.f64(_grid(g, shape, -6, -1))))
        xs += [_grid(g, shape, -12, 2, 0.1) for _ in range(W - 2)]
        residual = _grid(g, shape, -8, 0, 0.1)
    elif family == "eps":
        rms = torch.pow(10.0, torch.rand((T, 1), generator=g) * 2 - 4)
        xs = [(torch.randn(shape, generator=g) * rms / W ** 0.5).to(torch.bfloat16) for _ in range(W)]
        residual = (torch.randn(shape, generator=g) * rms / 2).to(torch.bfloat16)
        zero = torch.arange(T) % 5 == 3
        for x in xs + [residual]:
            x[zero] = 0
    elif family == "lamport":
        xs = [torch.randn(shape, generator=g).to(torch.bfloat16) for _ in range(W)]
        residual = torch.randn(shape, generator=g).to(torch.bfloat16)
        for x in xs:  # sentinel words in the inputs: (+0.0, -0.0) pairs
            w = x.view(torch.int32)
            w[torch.rand(w.shape, generator=g) < 0.2] = SENTINEL
        if W >= 2:  # positions whose sum cancels to zero under a -0.0 high half (see above)
            rows = torch.arange(T) % 3 == 0
            pick = (torch.rand((T, H // 2), generator=g) < 0.3) & rows[:, None]
            tiny = 2.0 ** -10
            for r, x in enumerate(xs):
                lo = torch.full((T, H // 2), tiny if r == 0 else (-tiny if r == 1 else 0.0))
                pair = torch.stack([lo, torch.full_like(lo, -0.0)], -1).to(torch.bfloat16)
                pw = pair.view(torch.int32).reshape(T, H // 2)
                x.view(torch.int32)[pick] = pw[pick]
    else:
        raise ValueError(family)
    return dict(xs=[x.contiguous() for x in xs], residual=residual.contiguous(), weight=weight, eps=eps)


# ---- one-GPU drivers -------------------------------------------------------------------------------
def _lib():
    import hpc
    return hpc._ffi


def nan_rows(T, H, guard, device="cuda"):
    """[T + 2 guard, H] bf16 of NaN: the call writes the middle T rows, the guards must stay NaN."""
    return torch.full((T + 2 * guard, H), float("nan"), dtype=torch.bfloat16, device=device)


def ht_c(x, residual, weight, eps, out, out_res, num_max_blocks, signal=None, peers=None,
         rank=0, world=1, num_tokens=None, stream=None):
    """hpc_fuse_allreduce_rmsnorm_high_throughput_p2p_async on raw pointers (P2P or W = 1)."""
    f = _lib()
    H = weight.numel()
    T = x.shape[0] if num_tokens is None else num_tokens
    pin = pout = None
    if peers is not None:
        pin = (ctypes.c_int64 * world)(*peers[0])
        pout = (ctypes.c_int64 * world)(*peers[1])
    f.check(f.lib.hpc_fuse_allreduce_rmsnorm_high_throughput_p2p_async(
        x.data_ptr(), None, residual.data_ptr(), weight.data_ptr(), out.data_ptr(), None,
        out_res.data_ptr(), None if signal is None else signal.data_ptr(), pin, pout, rank, world,
        num_max_blocks, eps, T, H, stream or f.stream_of(x)), "allreduce ht")


def ll_c(x, residual, weight, eps, out, out_res, ptrs, ws, flags, world, rank, protocol,
         num_max_blocks=0, num_tokens=None):
    f = _lib()
    T = x.shape[0] if num_tokens is None else num_tokens
    f.check(f.lib.hpc_fuse_allreduce_rmsnorm_low_latency_ex_async(
        world, rank, T, weight.numel(), ptrs.data_ptr(), ws.data_ptr(), None, flags.data_ptr(), 1,
        0, x.data_ptr(), residual.data_ptr(), weight.data_ptr(), eps, out_res.data_ptr(),
        out.data_ptr(), num_max_blocks, protocol, f.stream_of(x)), "allreduce ll")


def ll_buf_bytes(T, W, H, big):
    """Bytes per Lamport buffer: the reference tests' sizing (2 ceil(T/W) W rows of H per buffer),
    or one that also holds the one-shot image [T][W][H] with an odd number of 16-byte units."""
    ref = 2 * ox.ceil_div(T, W) * W * H * 2
    return max(ref, T * W * H * 2) + 16 * 37 if big else ref


def new_flags(buf_bytes, cur=0, device="cuda"):
    return torch.tensor([cur, (cur + 2) % 3, buf_bytes, 0, 0, 0, 0, 0, 0], dtype=torch.int32,
                        device=device)


class HtSim:
    """W ranks' input / output slices and signal pads of the high-throughput path on one device."""

    def __init__(self, xs, H, device="cuda"):
        self.W, self.H = len(xs), H
        self.ins = [x.to(device).contiguous() for x in xs]
        self.outs = [torch.full_like(self.ins[0], float("nan")) for _ in range(self.W)]
        self.pads = [torch.zeros(64, dtype=torch.int32, device=device) for _ in range(self.W)]
        self.signal = torch.tensor([p.data_ptr() for p in self.pads], dtype=torch.int64, device=device)

    def launch(self, rank, s, e, residual, weight, eps, out_res, num_max_blocks):
        """Rank `rank` reduces rows [s, e). Its pad's entry and exit words are set to 2^30 first:
        every simulated peer has already arrived and left, so no wait can block."""
        self.pads[rank][:32] = ARRIVED
        off = s * self.H * 2
        peers = ([b.data_ptr() + off for b in self.ins], [b.data_ptr() + off for b in self.outs])
        ht_c(self.ins[rank][s:], residual, weight, eps, self.outs[rank][s:], out_res, num_max_blocks,
             self.signal, peers, rank, self.W, num_tokens=e - s)


def ll_sim(xs, residual, weight, eps, rank, protocol, buf_bytes, out, out_res, cur=1,
           num_max_blocks=0, device="cuda"):
    """One launch of rank `rank` with W - 1 simulated peers and no multicast mapping. Returns
    (one_shot, own workspace, peer workspaces {p: int32}, flags). The rank's current buffer is
    pre-filled by oracle.allreduce_exact.ll_prefill; every other buffer and every peer's
    workspace starts as sentinel. out / out_res: [T, H] views the call writes."""
    W = len(xs)
    T, H = xs[0].shape
    one_shot, _ = ox.ll_protocol(T, W, H, buf_bytes, protocol)
    words = buf_bytes // 4
    sums = None if one_shot else ox.to_bf16(ox.emulate_sum(xs))
    img = ox.ll_prefill(T, W, H, rank, one_shot, xs, sums, words, POISON)
    own = torch.full((3 * words,), SENTINEL, dtype=torch.int32, device=device)
    own[cur * words:(cur + 1) * words] = torch.from_numpy(img).to(device)
    peers = {p: torch.full((3 * words,), SENTINEL, dtype=torch.int32, device=device)
             for p in range(W) if p != rank}
    ptrs = torch.tensor([own.data_ptr() if p == rank else peers[p].data_ptr() for p in range(W)],
                        dtype=torch.int64, device=device)
    flags = torch.tensor([cur, cur, buf_bytes, 0, 0, 0, 0, 0, 0], dtype=torch.int32, device=device)
    ll_c(xs[rank].to(device), residual.to(device), weight.to(device), eps, out, out_res, ptrs, own,
         flags, W, rank, protocol, num_max_blocks)
    return one_shot, own, peers, flags, sums
