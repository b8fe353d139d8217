#!/usr/bin/env python
"""Shape count of k_schur's SYRK on the seeded windows (synthetic.make_window(config, 0..7), cfg-2 by default), on the CPU.

Landmarks are sorted by (first, last) observing frame as the upload does and grouped into tiles of 32.  Per window and
solver round it prints: tiles, mean frame range u, how often the range changes from one tile to the next, the
multiply-adds inside the tile ranges (6x6 blocks of the lower triangle + the augmented row over 96 rows), those of the
landmarks' real tracks, the lane-FMA slots of the former one-lane-per-6x6-block mapping (6 warps, up to 8 column
splits per block pair, whole warps issue), and the DMMAs of the former frame-pair layout (u(u+1)/2 8x8 blocks x 24 k-steps;
fragment loads per DMMA for the one- and two-pair items the warps take), and the same for the packed layout k_schur
runs: the 6K pose columns in ceil(6K / 8) blocks of 8, one 8x8 block per pair of the blocks a tile's range touches,
the right-hand side formed in the Y build instead (no DMMA).

    python tools/schur_shapes.py [--config 2] [--windows 8]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from okvis_b200 import synthetic  # noqa: E402


def tracks(w):
    L = len(w.landmarks)
    vis = np.zeros(L, dtype=np.int64)
    np.bitwise_or.at(vis, w.obs["lm_idx"].astype(np.int64), np.left_shift(1, w.obs["pose_idx"].astype(np.int64)))
    first = np.array([int(v & -v).bit_length() - 1 if v else 32 for v in vis])
    last = np.array([int(v).bit_length() - 1 if v else 32 for v in vis])
    order = np.argsort(first * 32 + last, kind="stable")
    return vis[order], first[order], last[order]


def old_slots(u):
    """Lane-FMA slots the former mapping issued for one full tile of range u (6 warps of 32 lanes)."""
    n_act = u * (u + 1) // 2 + u
    ipw = (n_act + 5) // 6
    if ipw > 32:
        return ((n_act + 191) // 192) * 6 * 32 * 36 * 96
    ks = 1
    while 2 * ks <= 8 and 2 * ks * ipw <= 32:
        ks *= 2
    busy = sum(1 for w in range(6) if w * ipw < n_act)
    return busy * 32 * 36 * ((96 + ks - 1) // ks)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=2)
    ap.add_argument("--windows", type=int, default=8)
    args = ap.parse_args()
    tot = dict(tiles=0, u=0, changes=0, useful=0, real=0, old=0, dmma=0, loads=0, pdmma=0, ploads=0)
    for wi in range(args.windows):
        w = synthetic.make_window(args.config, wi)
        vis, first, last = tracks(w)
        prev = None
        for t in range(0, len(vis), 32):
            seen = vis[t:t + 32] != 0
            if not seen.any():
                continue
            fa, fb = int(first[t:t + 32][seen].min()), int(last[t:t + 32][seen].max())
            u = fb - fa + 1
            tot["tiles"] += 1
            tot["u"] += u
            tot["changes"] += (fa, fb) != prev
            prev = (fa, fb)
            tot["useful"] += 96 * (36 * u * (u + 1) // 2 + 6 * u)
            for v in vis[t:t + 32]:
                n = bin(int(v)).count("1")
                tot["real"] += 3 * (36 * n * (n + 1) // 2 + 6 * n)
            tot["old"] += old_slots(u)
            tot["dmma"] += 24 * u * (u + 1) // 2
            for il in range(u):        # row il: items of two pairs (3 loads per 2 DMMAs), a last single (1 load)
                tot["loads"] += 24 * (3 * ((il + 1) // 2) + ((il + 1) % 2))
            ub = (6 * fb + 5) // 8 - (6 * fa) // 8 + 1      # packed layout: blocks the range touches
            tot["pdmma"] += 24 * ub * (ub + 1) // 2
            for il in range(ub):
                tot["ploads"] += 24 * (3 * ((il + 1) // 2) + ((il + 1) % 2))
    n = args.windows
    print("windows: %d (cfg-%d, seeds 0..%d)" % (n, args.config, n - 1))
    print("tiles per window: %.1f, mean frame range u: %.2f" % (tot["tiles"] / n, tot["u"] / tot["tiles"]))
    print("frame-range changes per window per round: %.1f" % (tot["changes"] / n))
    print("per window per round, multiply-adds:")
    print("  inside the tile ranges        %6.2f M" % (tot["useful"] / n / 1e6))
    print("  of the real tracks            %6.2f M" % (tot["real"] / n / 1e6))
    print("  former lane-FMA slots issued  %6.2f M" % (tot["old"] / n / 1e6))
    print("  frame-pair layout: %d DMMA = %.2f M FMA-equivalents, %.2f fragment loads per DMMA" % (
        tot["dmma"] / n, tot["dmma"] * 256 / n / 1e6, tot["loads"] / tot["dmma"]))
    print("  packed layout: %d DMMA = %.2f M FMA-equivalents, %.2f fragment loads per DMMA (%+.1f %% DMMA)" % (
        tot["pdmma"] / n, tot["pdmma"] * 256 / n / 1e6, tot["ploads"] / tot["pdmma"], 100.0 * (tot["pdmma"] / tot["dmma"] - 1)))


if __name__ == "__main__":
    main()
