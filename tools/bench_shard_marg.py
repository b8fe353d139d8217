"""The per-frame cycle of a sliding cfg-5 window (20 keyframes, 4 cameras, 8000 landmarks at full size), unsharded on
one context and landmark-sharded over `world` contexts, as one JSON line.

Per slide step (tools/shard_slide_worker.py's Slide):
  optimize:     okb_optimize(max_iterations=10) on every rank;
  marginalize:  okb_window_marginalize of the oldest frame, its speed/bias, IMU term and finished landmarks on every rank;
  edits:        remove landmarks / frame, re-fix the first pose, add the next frame with its landmarks and observations
                (routed by owner), and the commit of them.
Each phase is timed on the host clock around work that ends in a synchronisation of every device used, so the
marginalisation is timed on its own.  world 2 and 4 run on one device (okb_shard_connect_local) -- which measures the
exchange and the redundant dense work, not multi-GPU scaling -- and across devices when there are enough of them.  The
card's name and power limit are read in the same run.  The first step is a warm-up and is left out of the medians.

    python tools/bench_shard_marg.py [--landmarks 8000] [--steps 6] [--worlds 1,2,4] [--out shard_marg.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from okvis_b200 import capi  # noqa: E402
from okvis_b200 import sharding  # noqa: E402
from shard_slide_worker import Slide, slide_problem  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def run(torch, full, w0, first_seen, world, devices, steps, iters):
    ctxs = [capi.Context(d, 1) for d in devices]
    try:
        if world > 1:
            capi.Context.shard_connect_local(ctxs, max_frames=len(w0.poses))
        s = Slide(list(enumerate(ctxs)), world, full, w0, first_seen)

        def sync():
            for d in sorted(set(devices)):
                torch.cuda.synchronize(d)

        rows = []
        for _ in range(steps):
            t0 = time.perf_counter()
            summ = s.optimize(iters)
            sync()
            t1 = time.perf_counter()
            parts = s.parts()
            est = sharding.merge_shard_results(s.L, parts)
            kw, cand = s.job(est)
            sync()
            t2 = time.perf_counter()
            s.marginalize(kw)
            sync()
            t3 = time.perf_counter()
            status = [int(g["status"][0]) for g in s.priors()]
            if any(status):
                raise SystemExit("world %d: marginalisation status %s" % (world, status))
            t4 = time.perf_counter()
            edited = s.edits(cand, est["poses"][1])
            for _, c in s.members:
                c.commit(0, 1)
            sync()
            t5 = time.perf_counter()
            s.follow(cand, *edited)
            faults = [c.shard_stats(0)["fault"] for c in ctxs] if world > 1 else [0]
            if any(faults) or any(x["termination"] == 6 for x in summ):
                raise SystemExit("world %d: a rank failed (%s)" % (world, faults))
            rows.append(dict(optimize_ms=1e3 * (t1 - t0), marginalize_ms=1e3 * (t3 - t2), edits_ms=1e3 * (t5 - t4),
                             iterations=summ[0]["iterations"], landmarks=len(kw["landmarks"])))
        timed = rows[1:] if len(rows) > 1 else rows
        med = {k: float(np.median([r[k] for r in timed])) for k in ("optimize_ms", "marginalize_ms", "edits_ms")}
        return dict(world=world, devices=list(devices), steps=rows, median=med)
    finally:
        for c in ctxs:
            c.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--landmarks", type=int, default=8000)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--iterations", type=int, default=10)
    ap.add_argument("--worlds", default="1,2,4")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_shard_marg needs a CUDA device")
    n_dev = torch.cuda.device_count()
    res = dict(card=card(), devices=n_dev, landmarks=args.landmarks, runs=[])
    print("card (name, power limit, max SM clock):", res["card"], flush=True)
    full, w0, first_seen = slide_problem(args.landmarks, extra=args.steps)
    for world in [int(x) for x in args.worlds.split(",")]:
        layouts = [[0] * world]
        if 1 < world <= n_dev:
            layouts.append(list(range(world)))
        for devices in layouts:
            r = run(torch, full, w0, first_seen, world, devices, args.steps, args.iterations)
            res["runs"].append(r)
            m = r["median"]
            print("world %d on devices %s: optimize(10) %.2f ms  marginalize %.3f ms  edits+commit %.3f ms  (median of %d steps, %s "
                  "landmarks marginalised)" % (world, devices, m["optimize_ms"], m["marginalize_ms"], m["edits_ms"], max(len(r["steps"]) - 1, 1),
                                               [x["landmarks"] for x in r["steps"]]), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
