"""Does splitting one batched solve into window groups on their own streams pay?  One JSON line.

Each group is a separate capi.Context on the same device (its own solver stream), holding a contiguous share of the
B cfg-2 windows; the whole batch is one more context of B windows.  `reset + optimize(10)` is timed three ways,
alternating, --reps each:
  whole:      the B-window context alone;
  split:      the G group contexts issued back to back (async calls, then the finishes);
  stagger_F:  as split, with group g's launch held back on its stream by g x F of one group round (a device-side
              sleep before its optimize), for each F of --stagger.
A group round is whole / (max_iterations + 1) / G: the round time of the whole batch scaled to one group's share.
Host clock around work that ends in a device synchronise, and CUDA events from a start event all streams wait on to
the last stream's end.  The summaries of every group are compared bit for bit with those of the whole batch.

    python tools/group_overlap_probe.py [--batch 528] [--groups 2] [--reps 5] [--stagger 0.5 1] [--out probe.json]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=528)
    ap.add_argument("--groups", type=int, nargs="+", default=[2])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--stagger", type=float, nargs="+", default=[0.5, 1.0])
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("group_overlap_probe needs a CUDA device")
    dev = torch.device("cuda", 0)
    B = args.batch
    res = dict(card=card(), batch=B, max_iterations=ITERS, reps=args.reps)
    print("card (name, power limit, max SM clock):", res["card"], flush=True)
    distinct = [synthetic.make_window(2, i) for i in range(args.distinct)]
    wins = [distinct[i % len(distinct)] for i in range(B)]

    whole = capi.Context(0, B)
    whole.upload_batch(0, wins)
    splits = {}
    for G in args.groups:
        bounds = [B * g // G for g in range(G + 1)]
        ctxs = []
        for g in range(G):
            c = capi.Context(0, bounds[g + 1] - bounds[g])
            c.upload_batch(0, wins[bounds[g]:bounds[g + 1]])
            ctxs.append(c)
        splits[G] = ctxs
    torch.cuda.synchronize(dev)

    # device-side delay: cycles of torch.cuda._sleep per millisecond
    s = torch.cuda.Stream(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(s):
        torch.cuda._sleep(1000)
        e0.record(s)
        torch.cuda._sleep(20_000_000)
        e1.record(s)
    torch.cuda.synchronize(dev)
    cycles_per_ms = 20_000_000 / e0.elapsed_time(e1)
    res["sleep_cycles_per_ms"] = cycles_per_ms

    def run(ctxs, delay_ms):
        """reset + optimize(ITERS) of every context; group g waits g * delay_ms on its stream first."""
        streams = [torch.cuda.ExternalStream(c.stream, device=dev) for c in ctxs]
        torch.cuda.synchronize(dev)
        start = torch.cuda.Event(enable_timing=True)
        ends = [torch.cuda.Event(enable_timing=True) for _ in ctxs]
        t0 = time.perf_counter()
        start.record(streams[0])
        for g, (c, st) in enumerate(zip(ctxs, streams)):
            if g:
                st.wait_event(start)
            if g and delay_ms > 0:
                with torch.cuda.stream(st):
                    torch.cuda._sleep(int(g * delay_ms * cycles_per_ms))
            c.reset(0, c.max_windows)
            c.optimize_async(0, c.max_windows, max_iterations=ITERS)
        out = []
        for c, st, e in zip(ctxs, streams, ends):
            out += c.optimize_finish(0, c.max_windows)
            e.record(st)
        torch.cuda.synchronize(dev)
        wall = time.perf_counter() - t0
        return 1e3 * wall, max(start.elapsed_time(e) for e in ends), out

    for _ in range(2):                            # warm-up: modules, graphs
        t_whole = run([whole], 0)[1]
        for G in args.groups:
            run(splits[G], 0)
    round_ms = t_whole / (ITERS + 1)
    variants = [("whole", [whole], 0.0)]
    for G in args.groups:
        variants.append(("split%d" % G, splits[G], 0.0))
        for f in args.stagger:
            variants.append(("split%d_stagger%g" % (G, f), splits[G], f * round_ms / G))
    for _, ctxs, d in variants:
        if d > 0:
            run(ctxs, d)
    times = {name: {"wall_ms": [], "event_ms": []} for name, _, _ in variants}
    summaries = {}
    for _ in range(args.reps):
        for name, ctxs, d in variants:
            w, e, out = run(ctxs, d)
            times[name]["wall_ms"].append(w)
            times[name]["event_ms"].append(e)
            summaries[name] = out
    strip = lambda x: {k: v for k, v in x.items() if k != "solve_time_s"}      # noqa: E731 (wall time, not a result)
    ref = [strip(x) for x in summaries["whole"]]
    res["round_ms_whole"] = round_ms
    for name, _, d in variants:
        t = times[name]
        res[name] = dict(delay_ms=d, event_ms_median=float(np.median(t["event_ms"])), event_ms_min=min(t["event_ms"]),
                         event_ms_max=max(t["event_ms"]), wall_ms_median=float(np.median(t["wall_ms"])),
                         event_ms_all=t["event_ms"], same_summaries=[strip(x) for x in summaries[name]] == ref)
        print("%-22s delay %.3f ms  events %7.2f ms [%7.2f, %7.2f]  wall %7.2f ms  same %s" % (
            name, d, res[name]["event_ms_median"], res[name]["event_ms_min"], res[name]["event_ms_max"],
            res[name]["wall_ms_median"], res[name]["same_summaries"]), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    whole.close()
    for ctxs in splits.values():
        for c in ctxs:
            c.close()


if __name__ == "__main__":
    main()
