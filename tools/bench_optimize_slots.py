"""Cost of solving a scattered set of resident windows, in one process, as one JSON line.

528 cfg-2 windows (synthetic.make_window(2, i)) are resident in one context.  A seeded set of 264 of them (ascending,
so it falls into runs of consecutive slots) is optimized with max_iterations=10 three ways:
  range:  okb_optimize over the contiguous slots 0..263 (the same batch size, for reference);
  set:    one okb_optimize_slots over the set;
  runs:   one okb_optimize_async per run of consecutive slots of the set, then one okb_optimize_finish per run.
Before every timed repetition the windows are restored, untimed, with okb_window_reset.  Host clock around work that
ends in a device synchronise; the three alternate in one run, best of --reps.  The set's summaries and estimates
are compared bit for bit with okb_optimize over a range of a second context that holds the same windows in the same
order; any difference fails the script.

    python tools/bench_optimize_slots.py [--windows 528] [--set 264] [--reps 5] [--out optimize_slots.json]
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


def runs_of(slots):
    runs = []
    for s in slots:
        if runs and runs[-1][0] + runs[-1][1] == s:
            runs[-1][1] += 1
        else:
            runs.append([s, 1])
    return runs


def estimates(ctx, slots):
    out = []
    for s in slots:
        d = ctx.download(s)
        out.append(b"".join(np.ascontiguousarray(d[k]).tobytes() for k in ("poses", "speed_bias", "landmarks", "quality")))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=528)
    ap.add_argument("--set", type=int, default=264)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_optimize_slots needs a CUDA device")
    n, m = args.windows, args.set
    res = dict(card=card(), windows=n, set_size=m, max_iterations=ITERS)
    print("card (name, power limit, max SM clock):", res["card"], flush=True)
    sync = torch.cuda.synchronize
    wins = [synthetic.make_window(2, i) for i in range(n)]
    ctx = capi.Context(0, n)
    ctx.upload_batch(0, wins)
    slots = sorted(int(x) for x in np.random.default_rng(args.seed).choice(n, m, replace=False))
    runs = runs_of(slots)
    res["n_runs"] = len(runs)

    def range_call():
        return ctx.optimize(0, m, max_iterations=ITERS)

    def set_call():
        return ctx.optimize_slots(slots, max_iterations=ITERS)

    def runs_call():
        for f, c in runs:
            ctx.optimize_async(f, c, max_iterations=ITERS)
        out = []
        for f, c in runs:
            out += ctx.optimize_finish(f, c)
        return out

    def timed(fn):
        ctx.reset(0, n)
        sync()
        l0 = ctx.kernel_launches
        t0 = time.perf_counter()
        s = fn()
        sync()
        return time.perf_counter() - t0, s, ctx.kernel_launches - l0

    for fn in (range_call, set_call, runs_call):       # warm-up: modules, graphs of every batch size
        timed(fn)
    t = {"range": [], "set": [], "runs": []}
    launches, iters = {}, {}
    for _ in range(args.reps):
        for name, fn in (("range", range_call), ("set", set_call), ("runs", runs_call)):
            dt, s, nl = timed(fn)
            t[name].append(dt)
            launches[name] = nl
            iters[name] = sum(x["iterations"] for x in s)
    # outputs: the set against a range of the same windows in the same order
    ctx.reset(0, n)
    got_s = set_call()
    got_e = estimates(ctx, slots)
    ctx.close()
    ref = capi.Context(0, m)
    ref.upload_batch(0, [wins[s] for s in slots])
    ref_s = ref.optimize(0, m, max_iterations=ITERS)
    ref_e = estimates(ref, range(m))
    ref.close()
    strip = lambda x: {k: v for k, v in x.items() if k != "solve_time_s"}      # noqa: E731 (wall time, not a result)
    same = got_e == ref_e and all(strip(a) == strip(b) for a, b in zip(got_s, ref_s))
    if not same:
        raise SystemExit("the set's outputs differ from a range holding the same windows in the same order")
    for name in t:
        res[name] = dict(ms=1e3 * min(t[name]), ms_all=[1e3 * x for x in t[name]], launches=launches[name],
                         iterations=iters[name], iterations_per_s=iters[name] / min(t[name]))
        print("%-5s %8.2f ms  (%s)  launches %d  iterations %d" % (
            name, res[name]["ms"], ", ".join("%.2f" % (1e3 * x) for x in t[name]), launches[name], iters[name]), flush=True)
    res["set_equals_range_bitwise"] = same
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
