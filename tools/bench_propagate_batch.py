"""Batched IMU propagation against a loop of the single call, in one process, as one JSON line.

Two workloads, at --sizes jobs (one job per session):
  frame: the prediction a VIO host makes per camera frame (ThreadedKFVio.cpp:416, Estimator::addStates): 52 samples per
         job (cfg-2's 0.25 s between frames at 200 Hz, plus the 5 ms overlaps), no covariance or Jacobian;
  imu:   the IMU-rate publisher (ThreadedKFVio.cpp:582): 2-3 samples per job, with covariance and Jacobian.
Each is timed alone and beside a solve: while an okb_optimize_async(max_iterations=10) of --solve cfg-2 windows is in
flight, the batch call and a loop of okb_imu_propagate over the same jobs are timed.  The single call runs on the
solver stream and so waits for the solve; the batch runs on its own stream.
Host clock around calls that end in a device synchronise; the ctypes arguments are built before the clock starts.
Loop and batch alternate in the same run, best of --reps, min-max spread reported.  In every repetition the batch's
outputs are compared bit for bit with the loop's; any difference fails the script.

    python tools/bench_propagate_batch.py [--sizes 1,8,132,528,2048] [--reps 5] [--solve 528] [--out prop.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from okvis_b200 import abi, capi, synthetic  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


class Jobs:
    """n seeded propagation jobs with their outputs, as an okb_propagate_job table and as single-call arguments."""

    def __init__(self, n, workload, seed):
        rng = np.random.default_rng(seed)
        self.prm = abi.make_imu_params()
        dt = 5_000_000
        want = workload == "imu"
        self.table = (abi.PropagateJob * n)()
        self.pose0, self.sb0, self.samples = [], [], []
        self.pose, self.sb = np.zeros((n, 7)), np.zeros((n, 9))
        self.P, self.F, self.n_used = np.zeros((n, 15, 15)), np.zeros((n, 15, 15)), np.zeros(n, np.int32)
        self.t = []
        for i in range(n):
            m = 52 if workload == "frame" else 2 + i % 2
            ts = 1_000_000_000 + int(rng.integers(0, dt)) + np.arange(m, dtype=np.int64) * dt
            s = np.zeros(m, abi.imu_sample_dtype)
            s["t_ns"] = ts
            s["gyro"] = rng.normal(0, 0.3, (m, 3))
            s["acc"] = rng.normal(0, 0.5, (m, 3)) + [0, 0, 9.81]
            t0, t1 = int(ts[0]) + dt // 4, int(ts[-1]) - dt // 3
            q = rng.normal(0, 1, 4)
            pose = np.concatenate([rng.uniform(-1, 1, 3), q / np.linalg.norm(q)])
            sb = np.concatenate([rng.normal(0, 0.5, 3), rng.normal(0, 0.01, 3), rng.normal(0, 0.05, 3)])
            self.samples.append(s)
            self.pose0.append(pose)
            self.sb0.append(sb)
            self.t.append((t0, t1))
            j = self.table[i]
            j.params, j.samples, j.n_samples, j.t0_ns, j.t1_ns = C.pointer(self.prm), s.ctypes.data, m, t0, t1
            j.pose = self.pose[i].ctypes.data_as(abi.c_double_p)
            j.speed_bias = self.sb[i].ctypes.data_as(abi.c_double_p)
            j.covariance = self.P[i].ctypes.data_as(abi.c_double_p) if want else None
            j.jacobian = self.F[i].ctypes.data_as(abi.c_double_p) if want else None
            j.n_used = self.n_used[i:].ctypes.data_as(C.POINTER(C.c_int32))
        self.n = n

    def reset(self):
        self.pose[:] = self.pose0
        self.sb[:] = self.sb0
        self.P[:] = 0
        self.F[:] = 0
        self.n_used[:] = 0

    def outputs(self):
        return b"".join(a.tobytes() for a in (self.pose, self.sb, self.P, self.F, self.n_used))

    def batch(self, ctx):
        rc = capi.lib().okb_imu_propagate_batch(ctx._h, self.n, self.table)
        if rc:
            raise SystemExit("okb_imu_propagate_batch failed: %d" % rc)

    def loop(self, ctx):
        f, h = capi.lib().okb_imu_propagate, ctx._h
        for j in self.table:
            rc = f(h, j.params, C.c_void_p(j.samples), j.n_samples, C.c_int64(j.t0_ns), C.c_int64(j.t1_ns), j.pose,
                   j.speed_bias, j.covariance, j.jacobian, j.n_used)
            if rc:
                raise SystemExit("okb_imu_propagate failed: %d" % rc)


def timed(jobs, fn, before=None, after=None):
    jobs.reset()
    if before:
        before()
    t0 = time.perf_counter()
    fn()
    dt = time.perf_counter() - t0
    if after:
        after()
    out = jobs.outputs()
    if (jobs.n_used <= 0).any():
        raise SystemExit("a job did not propagate")
    return dt, out


def stats(ts):
    return dict(best_ms=1e3 * min(ts), max_ms=1e3 * max(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,132,528,2048")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--solve", type=int, default=528, help="cfg-2 windows of the solve in flight")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_propagate_batch needs a CUDA device")
    res = dict(card=card(), solve_windows=args.solve, reps=args.reps, results={})
    print("card (name, power limit, max SM clock):", res["card"], flush=True)
    wins = [synthetic.make_window(2, i) for i in range(args.solve)]
    ctx = capi.Context(0, args.solve)
    ctx.upload_batch(0, wins)
    sync = torch.cuda.synchronize
    t_opt = []
    for _ in range(args.reps):
        ctx.reset(0, args.solve)
        sync()
        t0 = time.perf_counter()
        ctx.optimize(0, args.solve, max_iterations=10)
        t_opt.append(time.perf_counter() - t0)
    res["optimize10"] = stats(t_opt)
    print("optimize(10) of %d cfg-2 windows: %.2f ms" % (args.solve, 1e3 * min(t_opt)), flush=True)

    def solve_start():
        ctx.reset(0, args.solve)
        ctx.optimize_async(0, args.solve, max_iterations=10)

    def solve_end():
        ctx.optimize_finish(0, args.solve)

    for workload in ("frame", "imu"):
        for n in [int(s) for s in args.sizes.split(",")]:
            jobs = Jobs(n, workload, seed=1000 + n)
            timed(jobs, lambda: jobs.loop(ctx))         # warm-up; sizes the buffers
            timed(jobs, lambda: jobs.batch(ctx))
            sync()
            r = {}
            for mode, before, after in (("alone", None, None), ("beside_solve", solve_start, solve_end)):
                tl, tb = [], []
                for _ in range(args.reps):
                    d, ref = timed(jobs, lambda: jobs.loop(ctx), before, after)
                    tl.append(d)
                    d, got = timed(jobs, lambda: jobs.batch(ctx), before, after)
                    tb.append(d)
                    if got != ref:
                        raise SystemExit("%s n=%d %s: the batch's outputs differ from the single calls'" % (workload, n, mode))
                r[mode] = dict(loop=stats(tl), batch=stats(tb), speedup=min(tl) / min(tb))
                print("%-5s n=%4d %-12s loop %9.3f ms (max %9.3f)  batch %7.3f ms (max %7.3f)  x%.1f" % (
                    workload, n, mode, 1e3 * min(tl), 1e3 * max(tl), 1e3 * min(tb), 1e3 * max(tb), min(tl) / min(tb)), flush=True)
            res["results"]["%s_%d" % (workload, n)] = r
    ctx.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
