"""Throughput of the batched frontend against loops of the single calls, in one process, as one JSON line.

  detect: images/s of okb_detect_describe_batch at batch sizes 1..528 against okb_detect_describe called by 8 host
          threads, one per camera slot, over the same images (host clock around each call: packing, copies and
          kernels included; every figure is the best of 3 windows of >= 0.2 s of repeated calls), for the cfg-3 (15 px, <= 1000) and the shipped (40 px, <= 400) parameters;
  match:  pairs/s of okb_hamming_match_batch against a loop of okb_hamming_match(_gated), at the shipped shapes
          (~133 x 146, plain and 3D-2D gated), on the 300 x 450 gate test scene (3D-2D gated) and at cfg-3 (716 x 840);
  kernels: per-kernel device time of one 528-image batch from torch.profiler (a separate, profiled call).
Every timed batch's outputs are compared with the loop's; any difference fails the script.

    python tools/bench_frontend_batch.py [--reps 3] [--out frontend_batch.json]
"""
import argparse
import concurrent.futures as cf
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
from okvis_b200 import abi, capi, images  # noqa: E402
from gate_scene import gates, make_scene  # noqa: E402

CAM = abi.make_camera(abi.DIST_RADTAN, 752, 480, 458.654880721, 457.296696463, 367.215803962, 248.37534061,
                      (-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05))
PARAMS = {"cfg3": dict(uniformity_radius=15.0, max_keypoints=1000), "shipped": dict(uniformity_radius=40.0, max_keypoints=400)}
SIZES = [1, 8, 32, 132, 264, 528]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def best(f, reps, window=0.2):
    """Best over `reps` windows of the mean time per call; each window repeats f until it has run `window` seconds."""
    ts = []
    out = None
    for _ in range(reps):
        k, t0 = 0, time.perf_counter()
        while True:
            out = f()
            k += 1
            if time.perf_counter() - t0 >= window:
                break
        ts.append((time.perf_counter() - t0) / k)
    return min(ts), out


def same_det(a, b):
    return len(a[0]) == len(b[0]) and all(np.array_equal(a[0][f], b[0][f]) for f in a[0].dtype.names) and np.array_equal(a[1], b[1])


def same_match(a, b):
    return all(np.array_equal(a[k], b[k]) for k in ("topk", "pairs"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = dict(card=card(), detect={}, match={}, kernels_528={})
    print("card (name, power limit, max SM clock):", res["card"], flush=True)
    ctx = capi.Context(0, 1)
    pairs = [images.stereo_pair(seed=0x0B200 + 3000 + s) for s in range(16)]
    pool = [p[k] for p in pairs for k in (0, 1)]
    R = np.eye(3)
    ex = cf.ThreadPoolExecutor(8)
    for name, prm in PARAMS.items():
        res["detect"][name] = {}
        for n in SIZES:
            imgs = [pool[i % len(pool)] for i in range(n)]
            ctx.detect_describe_batch(imgs, [CAM] * n, [R] * n, **prm)            # warm-up: sizes the buffers

            def loop():
                futs = [ex.submit(lambda s: [ctx.detect_describe(imgs[i], CAM, R, cam_slot=s, **prm) for i in range(s, n, 8)], s)
                        for s in range(min(8, n))]
                per = [f.result() for f in futs]
                return [per[i % 8][i // 8] for i in range(n)]
            loop()
            t_loop, ref = best(loop, args.reps)
            t_batch, got = best(lambda: ctx.detect_describe_batch(imgs, [CAM] * n, [R] * n, **prm), args.reps)
            if not all(same_det(a, b) for a, b in zip(got, ref)):
                raise SystemExit("detect batch %s n=%d differs from the single calls" % (name, n))
            res["detect"][name][n] = dict(batch_images_per_s=n / t_batch, loop_images_per_s=n / t_loop, speedup=t_loop / t_batch,
                                          batch_ms=1e3 * t_batch)
            print("detect %-7s n=%3d  batch %8.0f img/s  loop %7.0f img/s  x%.1f" % (
                name, n, n / t_batch, n / t_loop, t_loop / t_batch), flush=True)
    sc = make_scene(0)
    g3, _ = gates(sc)
    rng = np.random.default_rng(1)
    idxA, idxB = rng.permutation(len(sc["A"]))[:133], rng.permutation(len(sc["B"]))[:146]
    big = rng.integers(0, 256, (840, 48), dtype=np.uint8)
    g3s = abi.make_match_gate(abi.GATE_3D2D, sc["kp_b"][idxB], sc["size_b"][idxB], proj_into_b=sc["proj"][idxA],
                              proj_uncertainty=sc["unc"][idxA])
    shapes = {"shipped_plain": dict(A=sc["A"][idxA], B=sc["B"][idxB]), "shipped_3d2d": dict(A=sc["A"][idxA], B=sc["B"][idxB], gate=g3s),
              "scene_3d2d_300x450": dict(A=sc["A"], B=sc["B"], gate=g3),
              "cfg3_plain": dict(A=big[:716], B=big[rng.permutation(840)])}
    for name, job in shapes.items():
        res["match"][name] = {}
        for n in SIZES:
            def loop():
                if "gate" in job:
                    return [ctx.hamming_match_gated(job["A"], job["B"], job["gate"]) for _ in range(n)]
                return [ctx.hamming_match(job["A"], job["B"]) for _ in range(n)]
            jobs = [ctx.make_match_job(**job) for _ in range(n)]
            ctx.hamming_match_batch(jobs, 48)
            t_loop, ref = best(loop, args.reps)
            t_batch, got = best(lambda: ctx.hamming_match_batch(jobs, 48), args.reps)
            if not all(same_match(a, b) for a, b in zip(got, ref)):
                raise SystemExit("match batch %s n=%d differs from the single calls" % (name, n))
            res["match"][name][n] = dict(batch_pairs_per_s=n / t_batch, loop_pairs_per_s=n / t_loop, speedup=t_loop / t_batch)
            print("match  %-18s n=%3d  batch %8.0f pairs/s  loop %7.0f pairs/s  x%.1f" % (
                name, n, n / t_batch, n / t_loop, t_loop / t_batch), flush=True)
    # where a 528-image batch spends its device time (profiled call, not used for the rates above)
    import torch
    from torch.profiler import ProfilerActivity, profile
    imgs = [pool[i % len(pool)] for i in range(528)]
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        ctx.detect_describe_batch(imgs, [CAM] * 528, [R] * 528, **PARAMS["cfg3"])
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        dt = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
        if dt and ("k_" in ev.key or "Memcpy" in ev.key or "Memset" in ev.key):
            res["kernels_528"][ev.key[:60]] = dt / 1e3
    for k, v in sorted(res["kernels_528"].items(), key=lambda kv: -kv[1]):
        print("  528-image batch (cfg-3): %-60s %8.3f ms" % (k, v))
    ctx.close()
    ex.shutdown()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
