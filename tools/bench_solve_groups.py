"""Cost of a batched solve split into window groups (okb_set_solve_groups), as one JSON line.

For each batch size B of --batches, B cfg-2 windows (synthetic.make_window(2, i % --distinct), as bench.py fills its
batch) are resident in one context, and `reset + optimize(10)` is timed with each forced group count of --groups and
with the automatic choice (0), alternating, --reps each.  Two launch modes are timed: stream launches (profiling on,
as in bench.py's timed region) and the captured CUDA graph (profiling off).  Device time from CUDA events on the
context stream; the host clock around work that ends in a device synchronise is reported beside it.  Every group
count's summaries and downloaded estimates are compared bit for bit with one group's; any difference fails the script.

    python tools/bench_solve_groups.py [--batches 132 264 528 1056] [--groups 1 2 3 4] [--reps 5] [--out groups.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from okvis_b200 import capi, synthetic  # noqa: E402

ITERS = 10


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def outputs(ctx, B):
    strip = lambda x: {k: v for k, v in x.items() if k != "solve_time_s"}      # noqa: E731 (wall time, not a result)
    summ = [strip(s) for s in ctx.optimize_finish(0, B)]
    est = b"".join(np.ascontiguousarray(d[k]).tobytes() for d in (ctx.download(i) for i in range(B))
                   for k in ("poses", "speed_bias", "landmarks", "quality"))
    return summ, est


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[132, 264, 528, 1056])
    ap.add_argument("--groups", type=int, nargs="+", default=[1, 2, 3, 4])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_solve_groups needs a CUDA device")
    dev = torch.device("cuda", 0)
    res = dict(card=card(), max_iterations=ITERS, reps=args.reps, batches={})
    print("card (name, power limit, max SM clock):", res["card"], flush=True)
    distinct = [synthetic.make_window(2, i) for i in range(args.distinct)]
    choices = list(dict.fromkeys([1] + list(args.groups) + [0]))      # one group first: the reference outputs
    for B in args.batches:
        ctx = capi.Context(0, B)
        ctx.upload_batch(0, [distinct[i % len(distinct)] for i in range(B)])
        stream = torch.cuda.ExternalStream(ctx.stream, device=dev)

        def run(G, profile):
            ctx.set_solve_groups(G)
            ctx.profile_enable(profile)
            torch.cuda.synchronize(dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record(stream)
            ctx.reset(0, B)
            ctx.optimize_async(0, B, max_iterations=ITERS)
            e1.record(stream)
            torch.cuda.synchronize(dev)
            wall = time.perf_counter() - t0
            out = outputs(ctx, B)
            launches = None
            if profile:
                p = ctx.profile_read()
                launches = (p["landmarks_launches"], p["solve_launches"])
            return e0.elapsed_time(e1), 1e3 * wall, out, launches

        modes = (("stream", True), ("graph", False))
        for G in choices:                          # warm-up: modules, graphs
            for _, prof in modes:
                run(G, prof)
        t = {(m, G): ([], []) for m, _ in modes for G in choices}
        ref, same, prof_launches = {}, {}, {}
        for _ in range(args.reps):
            for G in choices:
                for m, prof in modes:
                    ev, wall, out, pl = run(G, prof)
                    t[(m, G)][0].append(ev)
                    t[(m, G)][1].append(wall)
                    ref.setdefault(m, out)
                    same[(m, G)] = same.get((m, G), True) and out == ref[m]
                    if pl is not None:
                        prof_launches[G] = pl
        ctx.set_solve_groups(0)
        row = {}
        for (m, G), (ev, wall) in t.items():
            row["%s_G%d" % (m, G)] = dict(event_ms_median=float(np.median(ev)), event_ms_min=min(ev), event_ms_max=max(ev),
                                         wall_ms_median=float(np.median(wall)), same_as_G1=same[(m, G)])
            print("B %5d %-6s G %d  events %7.2f ms [%7.2f, %7.2f]  wall %7.2f ms  same %s" % (
                B, m, G, np.median(ev), min(ev), max(ev), np.median(wall), same[(m, G)]), flush=True)
        row["profile_launches"] = {str(G): v for G, v in prof_launches.items()}
        res["batches"][str(B)] = row
        ctx.close()
        if not all(same.values()):
            print(json.dumps(res))
            raise SystemExit("B = %d: outputs differ between group counts" % B)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
