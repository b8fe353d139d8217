"""Times okb_ransac_2d2d_batch at 1 / 132 / 528 sessions shaped like cfg 2 (two cameras, about 250 correspondences
each, 10 % injected wrong associations, a 30 cm baseline, pose initialisation on) against a loop of single-job calls
over the same sessions, both through Context.ransac_2d2d_batch.  Times are a host clock around the synchronising call
(the binding's job packing, the H2D copy, launch and D2H copy), the median over the repetitions.  There is no CPU
comparison: the reference's solvers (OpenGV) are not available.  Prints the card name and power limit from the same
run, and one JSON line; --out also writes that line to a file."""
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
import ransac2d2d_scene as S  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", default="1,132,528")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("card:", q)
    pool = [S.make_scene(500 + i, abi.DIST_RADTAN, 2, "large", 0.1) for i in range(8)]
    rows = []
    for n in [int(x) for x in args.sessions.split(",")]:
        ctx = capi.Context(0, n)
        for s in range(n):
            S.load(ctx, s, pool[s % len(pool)])
        jobs = [dict(S.job(pool[s % len(pool)], 1000 + s, initialize_pose=True), win=s) for s in range(n)]
        got = ctx.ransac_2d2d_batch(jobs)          # warm-up (module load, buffers)
        assert all(g["ret"] > 10 for g in got)
        tb, tl = [], []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            ctx.ransac_2d2d_batch(jobs)
            tb.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            for j in jobs:
                ctx.ransac_2d2d_batch([j])
            tl.append(time.perf_counter() - t0)
        b_ms, l_ms = 1e3 * float(np.median(tb)), 1e3 * float(np.median(tl))
        rows.append(dict(sessions=n, batch_call_ms=round(b_ms, 4), single_call_loop_ms=round(l_ms, 4)))
        print("sessions %4d  batch call %.3f ms  loop of single calls %.3f ms (medians of %d)" % (n, b_ms, l_ms, args.reps))
        ctx.close()
    line = json.dumps(dict(card=q, rows=rows))
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
