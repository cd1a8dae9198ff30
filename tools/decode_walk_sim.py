"""Model of the rotated bin walk of the decode kernels (csrc/decode_common.cuh, restated in
oracle/decode_walk.py): for every position on the per-head task line, at which step do the CTAs
that own that position for the different kv heads process it? CPU only.

    python tools/decode_walk_sim.py [--batch 64] [--ctx 8192] [--heads 8] [--ctas 132] [--mpl 64]

Prints the spread (max - min step over the heads) with and without the rotation. At the C2 shape the
rotation brings 95 % of the positions to spread 0 (the rest belong to bins that straddle a head
boundary); front to back the mean spread is ~190 steps of ~0.85 us.
"""
import argparse
import collections
import statistics
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from oracle import decode_walk as dw  # noqa: E402


def spreads(lens, heads, ctas, rotate, min_process_len=64):
    """Spread of every task-line position, and the bin size P, for the walk of the task map that
    oracle.taskmap.assign builds for `lens` (the new token included)."""
    tm = dw.task_map(lens, ctas, heads, 1, min_process_len)
    tb = int(tm[0, 6])
    first = [0]
    for n in lens:
        first.append(first[-1] + (n + dw.TILE - 1) // dw.TILE)
    at = collections.defaultdict(list)
    for w in dw.walk(tm, len(lens), heads, rotate=rotate):
        t = 0
        for s in w["segs"]:
            te = s["tiles"] if s["te"] < 0 else s["te"]
            for tile in range(s["tb"], te):
                at[first[s["b"]] + s["start"] // dw.TILE + tile].append(t)
                t += 1
    return [max(v) - min(v) for v in at.values()], int(tm[0, 0]) - 1, tb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--ctx", type=int, default=8192)
    ap.add_argument("--heads", type=int, default=8)
    ap.add_argument("--ctas", type=int, default=132)
    ap.add_argument("--mpl", type=int, default=64)
    a = ap.parse_args()
    for rot in (False, True):
        s, p, tb = spreads([a.ctx] * a.batch, a.heads, a.ctas, rot, a.mpl)
        print(f"rotate={rot}: tiles/head {tb}, tiles/bin {p}: spread max {max(s)}, mean "
              f"{statistics.mean(s):.1f}, positions with spread 0: {sum(1 for v in s if v == 0) / len(s):.3f}")


if __name__ == "__main__":
    main()
