"""Times okb_ransac_3d2d_batch at 1 / 132 / 528 sessions shaped like cfg 2 (two cameras, about 400 keypoints each, 10 %
injected wrong associations) against a loop of single-job calls over the same sessions, both through
Context.ransac_3d2d_batch.  Times are a host clock around the synchronising call (the binding's job packing, the H2D
copy, launch and D2H copy), the median over the repetitions.  There is no CPU
comparison: the reference's solver (OpenGV) is not available.  Prints the card name and power limit from the same run,
and one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from okvis_b200 import abi, capi  # noqa: E402
import ransac_scene as S  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", default="1,132,528")
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("card:", q)
    pool = [S.make_scene(500 + i, abi.DIST_RADTAN, 2, 0.1) for i in range(8)]
    n_kp = max(len(e["lm"]) for sc in pool for e in sc["store"].values())
    rows = []
    for n in [int(x) for x in args.sessions.split(",")]:
        ctx = capi.Context(0, n)
        for s in range(n):
            S.load(ctx, s, pool[s % len(pool)], n_kp)
        jobs = [dict(win=s, feat_slot=S.FEAT, n_cams=2, seed=1000 + s) for s in range(n)]
        got = ctx.ransac_3d2d_batch(jobs)          # warm-up (module load, buffers)
        assert all(g["n_inliers"] >= 10 for g in got)
        tb, tl = [], []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            ctx.ransac_3d2d_batch(jobs)
            tb.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            for j in jobs:
                ctx.ransac_3d2d_batch([j])
            tl.append(time.perf_counter() - t0)
        b_ms, l_ms = 1e3 * float(np.median(tb)), 1e3 * float(np.median(tl))
        rows.append(dict(sessions=n, batch_call_ms=round(b_ms, 4), single_call_loop_ms=round(l_ms, 4)))
        print("sessions %4d  batch call %.3f ms  loop of single calls %.3f ms (medians of %d)" % (n, b_ms, l_ms, args.reps))
        ctx.close()
    print(json.dumps(dict(card=q, rows=rows)))


if __name__ == "__main__":
    main()
