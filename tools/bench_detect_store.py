"""Detection into the windows' feature stores, three ways, for 1, 132 and 528 stereo sessions of 752x480 images
(okvis_b200.images), at the cfg-3 (15 px, <= 1000) and the shipped (40 px, <= 400) parameters:

  (a) store: one okb_detect_describe_store_batch for every session's frame (keypoints back, descriptors stay on the device);
  (b) batch: okb_detect_describe_batch, okb_window_set_features per image, okb_window_commit;
  (c) loop:  okb_detect_describe per image plus okb_window_set_features, then okb_window_commit (the C++ mirror's path
             before the store form).

Each figure is the median over --reps of a host clock around the path, ending in a device synchronisation, after one
untimed run.  H2D / D2H bytes are computed from the shapes and the keypoint counts.  (a) and (b) must leave identical
store contents (okb_debug_features on every image) and identical keypoints; any difference fails the script.  The card's
name and power limit are read in the same run.

    python tools/bench_detect_store.py [--reps 10] [--out detect_store.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from okvis_b200 import abi, capi, images, synthetic  # noqa: E402

CAM = abi.make_camera(abi.DIST_RADTAN, 752, 480, 458.654880721, 457.296696463, 367.215803962, 248.37534061,
                      (-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05))
PARAMS = {"cfg3": dict(uniformity_radius=15.0, max_keypoints=1000), "shipped": dict(uniformity_radius=40.0, max_keypoints=400)}
SESSIONS = [1, 132, 528]
DESC = 48
FE_IMAGE, STORE_DEST, CMD_HEADER = 184, 48, 16     # bytes of the detector's per-image table entries and a command header


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    lines = q.stdout.strip().splitlines()
    return lines[0] if lines else "unknown"


def median_time(f, reps):
    import torch
    f()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def pad8(n):
    return (n + 7) // 8 * 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = dict(card=card(), runs={})
    print("card (name, power limit):", res["card"], flush=True)
    pool = [p[k] for p in (images.stereo_pair(seed=0x0B200 + 3000 + s) for s in range(16)) for k in (0, 1)]
    R = np.eye(3)
    w = synthetic.make_window(1, 0)
    for n in SESSIONS:
        ctx = capi.Context(0, n)
        maxk_all = max(p["max_keypoints"] for p in PARAMS.values())
        for s in range(n):
            ctx.reserve(s, len(w.poses), len(w.landmarks), len(w.obs), len(w.imu_samples))
            ctx.reserve_features(s, 3, 2, maxk_all, DESC)
            ctx.upload(s, w)
        imgs = [pool[(2 * s + c) % len(pool)] for s in range(n) for c in range(2)]
        pixels = sum(im.size for im in imgs)
        for name, prm in PARAMS.items():
            prm = dict(prm, desc_bytes=DESC)
            maxk = prm["max_keypoints"]
            jobs = [dict(imgs=imgs[2 * s:2 * s + 2], cams=[CAM, CAM], R_CWs=[R, R], win=s, feat_slot=0, want_desc=False) for s in range(n)]
            out = {}

            def store():
                out["a"] = ctx.detect_describe_store_batch(jobs, **prm)

            def batch(slot=1):
                got = ctx.detect_describe_batch(imgs, [CAM] * (2 * n), [R] * (2 * n), **prm)
                for i, (kp, desc) in enumerate(got):
                    ctx.set_features(i // 2, slot, i % 2, kp, desc)
                ctx.commit(0, n)
                out["b"] = got

            def loop():
                got = [ctx.detect_describe(im, CAM, R, **prm) for im in imgs]
                for i, (kp, desc) in enumerate(got):
                    ctx.set_features(i // 2, 2, i % 2, kp, desc)
                ctx.commit(0, n)
                out["c"] = got

            t_a = median_time(store, args.reps)
            t_b = median_time(batch, args.reps)
            t_c = median_time(loop, max(1, args.reps // 2 if n > 132 else args.reps))
            kps = [out["b"][i][0] for i in range(2 * n)]
            for i in range(2 * n):
                a = out["a"][i // 2][i % 2][0]
                if a.tobytes() != kps[i].tobytes() or out["c"][i][0].tobytes() != kps[i].tobytes():
                    raise SystemExit("%s n=%d: keypoints of image %d differ between the paths" % (name, n, i))
                ea, eb = ctx.debug_features(i // 2, 0, i % 2), ctx.debug_features(i // 2, 1, i % 2)
                if ea["n"] != eb["n"] or any(ea[f].tobytes() != eb[f].tobytes() for f in ("kp", "size", "desc", "lm_slot", "observed")):
                    raise SystemExit("%s n=%d: store entry of image %d differs between (a) and (b)" % (name, n, i))
            n_img, n_kp = 2 * n, sum(len(k) for k in kps)
            set_feat = sum(CMD_HEADER + 24 * len(k) + pad8(4 * len(k)) + pad8(len(k)) + pad8(DESC * len(k)) for k in kps)
            bytes_ = {
                "a": dict(h2d=pixels + n_img * (FE_IMAGE + STORE_DEST), d2h=n_img * (16 + 24 * maxk)),
                "b": dict(h2d=pixels + n_img * FE_IMAGE + set_feat, d2h=n_img * (16 + (24 + DESC) * maxk)),
                "c": dict(h2d=pixels + n_img * FE_IMAGE + set_feat, d2h=n_img * (16 + (24 + DESC) * maxk)),
            }
            r = dict(images=n_img, keypoints=n_kp, ms=dict(a_store=1e3 * t_a, b_batch_set_features=1e3 * t_b, c_loop_set_features=1e3 * t_c),
                     images_per_s=dict(a=n_img / t_a, b=n_img / t_b, c=n_img / t_c), bytes=bytes_)
            res["runs"]["%s_%d" % (name, n)] = r
            print("%-7s sessions=%3d images=%4d  (a) %8.2f ms  (b) %8.2f ms  (c) %8.2f ms   H2D a/b %.1f/%.1f MB  D2H a/b %.1f/%.1f MB" % (
                name, n, n_img, 1e3 * t_a, 1e3 * t_b, 1e3 * t_c, bytes_["a"]["h2d"] / 1e6, bytes_["b"]["h2d"] / 1e6,
                bytes_["a"]["d2h"] / 1e6, bytes_["b"]["d2h"] / 1e6), flush=True)
        ctx.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
