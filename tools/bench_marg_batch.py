"""Batched device marginalisation against a loop of the single call, in one process, as one JSON line.

For 132 and 528 cfg-2 windows (synthetic.make_window(2, i), reserved with max_marg_dim 80), each job marginalises
frame 0 (pose + speed/bias, IMU term 0, the speed/bias prior and the landmarks frame 0 ends), as a VIO host does once
per frame:
  loop:     okb_window_marginalize over all slots;
  batch:    one okb_window_marginalize_batch over the same slots;
  optimize: okb_optimize(max_iterations=10) of the same windows, for the marginalisation's share of a frame.
Host clock around work that ends in a device synchronise; loop and batch alternate in the same run, best of --reps.
Before every timed repetition the pre-marginalisation state is restored, untimed (okb_window_reset does not restore
the prior): upload_batch + optimize(5).  Every timed batch's priors are compared bit for bit with the loop's; any
difference fails the script.  k_marginalize's device time comes from torch.profiler in a separate, profiled pass.

    python tools/bench_marg_batch.py [--sizes 132,528] [--reps 3] [--out marg_batch.json]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from okvis_b200 import abi, capi, synthetic  # noqa: E402

P, SB = abi.BLOCK_POSE, abi.BLOCK_SPEED_BIAS


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def oldest_frame_job(w):
    L = len(w.landmarks)
    last, first = np.full(L, -1), np.full(L, 99)
    np.maximum.at(last, w.obs["lm_idx"], w.obs["pose_idx"])
    np.minimum.at(first, w.obs["lm_idx"], w.obs["pose_idx"])
    lms = np.nonzero((first == 0) & (last <= 2))[0].astype(np.uint32)
    sbp = [0] if len(w.sb_priors) and int(w.sb_priors["sb_idx"][0]) == 0 else []
    return abi.make_marg_job([P, SB, P, SB, P], [0, 0, 1, 1, 2], [-1] * 5, [1, 1, 0, 0, 0], imu_terms=[0], sb_priors=sbp,
                             landmarks=lms)


def priors(ctx, n):
    out = []
    for i in range(n):
        m = ctx.download_marg(i)
        out.append(b"".join(np.ascontiguousarray(m[k]).tobytes() for k in ("block_kind", "block_idx", "x0", "J", "e0", "H", "b0", "status")))
    return out


def kernel_ms(torch, fn):
    """Total device time and launch count of k_marginalize inside fn (profiled; other kernels are left out)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    total, count = 0.0, 0
    for ev in prof.key_averages():
        if "k_marginalize" in ev.key:
            total += (getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)) / 1e3
            count += ev.count
    return total, count


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="132,528")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_marg_batch needs a CUDA device")
    res = dict(card=card(), sms=torch.cuda.get_device_properties(0).multi_processor_count, sizes={})
    print("card (name, power limit, max SM clock):", res["card"], flush=True)
    sync = torch.cuda.synchronize
    for n in [int(s) for s in args.sizes.split(",")]:
        wins = [synthetic.make_window(2, i) for i in range(n)]
        ctx = capi.Context(0, n)
        for i, w in enumerate(wins):
            ctx.reserve(i, len(w.poses), len(w.landmarks), len(w.obs), len(w.imu_samples), 80)
        descs = ctx.make_descs(wins)
        jobs = [oldest_frame_job(w) for w in wins]

        def restore():
            ctx.upload_batch(0, wins, descs=descs)
            ctx.optimize(0, n, max_iterations=5)
            sync()

        def loop():
            for i in range(n):
                ctx.marginalize(i, jobs[i])

        def batch():
            ctx.marginalize_batch(0, jobs)

        def timed(fn):
            restore()
            t0 = time.perf_counter()
            fn()
            sync()
            return time.perf_counter() - t0

        timed(loop)             # warm-up: scratch, batch buffer, modules
        timed(batch)
        t_loop, t_batch, ref = [], [], None
        for _ in range(args.reps):
            t_loop.append(timed(loop))
            got_loop = priors(ctx, n)
            t_batch.append(timed(batch))
            got_batch = priors(ctx, n)
            if got_batch != got_loop:
                raise SystemExit("n=%d: the batch's priors differ from the single calls'" % n)
            if ref is not None and got_loop != ref:
                raise SystemExit("n=%d: the single calls are not reproducible" % n)
            ref = got_loop
        if any(int(np.frombuffer(p[-16:], np.int32)[0]) != 0 for p in ref):
            raise SystemExit("n=%d: a job reported a device error" % n)
        t_opt, iters = [], 0
        for _ in range(args.reps):
            ctx.upload_batch(0, wins, descs=descs)
            sync()
            t0 = time.perf_counter()
            s = ctx.optimize(0, n, max_iterations=10)
            t_opt.append(time.perf_counter() - t0)
            iters = sum(x["iterations"] for x in s)
        # the restore runs inside the profiled region: the profiler can miss the first kernels after it starts
        k_batch, c_batch = kernel_ms(torch, lambda: (restore(), batch()))
        k_loop, c_loop = kernel_ms(torch, lambda: (restore(), loop()))
        ctx.close()
        single_kernel = k_loop / max(c_loop, 1)
        r = dict(loop_ms=1e3 * min(t_loop), batch_ms=1e3 * min(t_batch), speedup=min(t_loop) / min(t_batch),
                 optimize10_ms=1e3 * min(t_opt), optimize10_iterations=iters,
                 batch_share_of_frame=min(t_batch) / (min(t_batch) + min(t_opt)),
                 loop_share_of_frame=min(t_loop) / (min(t_loop) + min(t_opt)),
                 k_marginalize_batch_ms=k_batch, k_marginalize_batch_launches=c_batch,
                 k_marginalize_single_ms=single_kernel, k_marginalize_loop_total_ms=k_loop, k_marginalize_loop_launches=c_loop,
                 waves=math.ceil(n / res["sms"]), waves_times_single_ms=math.ceil(n / res["sms"]) * single_kernel,
                 landmarks_per_job=float(np.mean([j.n_landmarks for j in jobs])))
        res["sizes"][n] = r
        print("n=%3d  loop %8.2f ms  batch %7.2f ms  x%.1f  optimize(10) %7.2f ms  k_marginalize: batch %.2f ms, single %.3f ms "
              "(%d waves -> %.2f ms)" % (n, r["loop_ms"], r["batch_ms"], r["speedup"], r["optimize10_ms"], k_batch, single_kernel,
                                        r["waves"], r["waves_times_single_ms"]), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
