"""The frontend calls on the feature store of a cfg-5 shaped window (20 keyframes, 4 cameras, 8000 landmarks at full
size), unsharded on one context and landmark-sharded over `world` contexts, as one JSON line.

The window is tools/shard_slide_worker.py's first window; its feature store holds, per frame and camera, the keypoints of
the frame's observations (the landmark's descriptor with a bit flipped) and 30 unrelated ones, the newest frame untracked.
Each rep runs one frame's sequence on the newest frame: detect into a spare feature slot (4 images), the 3D-2D rounds
against the 3 previous frames and the stereo pair, a 2D-2D round, RANSAC 3D-2D, the keyframe decision and stereo
initialisation (the warm-up rep tracks the frame; the timed reps run the same calls on the tracked frame).  Every
call is timed on the host clock around the call, which returns after its device work; the ranks of a sharded window
make each call at once from one host thread each, and the call's time is until the last rank returns.  Medians over
--reps after one warm-up rep.  world 2 and 4 run on one device (okb_shard_connect_local): that measures the landmark
exchange and the redundant work of every rank, not multi-GPU scaling.  The card's name and power limit are read in the
same run.

    python tools/bench_shard_frontend.py [--landmarks 8000] [--reps 10] [--worlds 1,2,4] [--out shard_frontend.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from okvis_b200 import capi, images  # noqa: E402
from shard_slide_worker import Slide, slide_problem  # noqa: E402

CALLS = ("detect", "track", "match2d2d", "ransac", "keyframe", "stereo")
N_KP, DESC = 384, 48
R_LIST = [np.eye(3), np.array([[0.9950, 0.0, -0.0998], [0.0198, 0.9801, 0.1977], [0.0978, -0.1987, 0.9752]])]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def frame_features(full, k, cam, base, n_max, tracked):
    """Keypoints of generated frame k in camera `cam`: its observations (descriptor of the landmark, a bit flipped) and
    30 unrelated ones; landmark slots set when the frame is already tracked.  ((x, y, size) [n][3], descriptors,
    landmark slots, observed flags), as okb_window_set_features takes them."""
    rng = np.random.default_rng(1000 * k + cam)
    o = full.obs[(full.obs["pose_idx"] == k) & (full.obs["cam_idx"] == cam)]
    lm = o["lm_idx"].astype(np.int32)
    desc = base[lm].copy()
    if len(lm):
        desc[np.arange(len(lm)), rng.integers(0, desc.shape[1], len(lm))] ^= np.uint8(1) << rng.integers(0, 8, len(lm)).astype(np.uint8)
    W, H = int(full.cameras[cam]["width"]), int(full.cameras[cam]["height"])
    n_x = 30
    kp = np.concatenate([o["z"], rng.uniform([0, 0], [W, H], (n_x, 2))])
    desc = np.concatenate([desc, rng.integers(0, 256, (n_x, base.shape[1]), dtype=np.uint8)])
    lm = np.concatenate([lm, -np.ones(n_x, np.int32)])
    order = rng.permutation(len(lm))[:n_max]
    kp, desc, lm = kp[order], desc[order], lm[order]
    kps = np.stack([kp[:, 0], kp[:, 1], rng.uniform(6.0, 14.0, len(lm))], 1).astype(np.float32).astype(np.float64)
    if not tracked:
        return kps, desc, -np.ones(len(lm), np.int32), np.zeros(len(lm), np.uint8)
    return kps, desc, lm, (lm >= 0).astype(np.uint8)


def camera_images(seed, cams):
    """One seeded textured view per camera (the stereo pair's two images, then further seeds), as detect jobs take them."""
    out = []
    for c in range(len(cams)):
        left, right = images.stereo_pair(seed=seed + c // 2)
        out.append(left if c % 2 == 0 else right)
    return dict(imgs=out, cams=list(cams), R_CWs=[R_LIST[c % 2] for c in range(len(cams))])


def load(s, full, w0, F):
    """Fills the feature store of every member of Slide `s`: frames 0..K-1 in feature slots 0..K-1, the newest untracked."""
    K, L, C = len(w0.poses), len(w0.landmarks), len(w0.cameras)
    base = np.random.default_rng(7).integers(0, 256, (L, DESC), dtype=np.uint8)
    for k in range(K):
        for cam in range(C):
            s.edit("set_features", k, cam, *frame_features(full, k, cam, base, N_KP, tracked=k < K - 1))
        for _, c in s.members:
            c.commit(0, 1)
    s.edit("set_landmark_initialized", np.arange(L), np.any(w0.landmarks != 0, axis=1).astype(np.uint8))
    for _, c in s.members:
        c.commit(0, 1)


def jobs(w0, F):
    K, C = len(w0.poses), len(w0.cameras)
    B = K - 1
    return dict(
        detect=[dict(camera_images(0x0B200 + 500, w0.cameras), win=0, feat_slot=F - 1)],
        track=[dict(win=0, pose_b=B, sb_b=B, feat_slot_b=B, rounds=[(B - a, c, c) for a in (1, 2, 3) for c in range(C)] + [(B, 0, 1), (B, 1, 0)])],
        match2d2d=[dict(win=0, pose_a=B - 1, feat_slot_a=B - 1, cam_a=0, pose_b=B, feat_slot_b=B, cam_b=0, sb_current=B)],
        ransac=[dict(win=0, feat_slot=B, n_cams=C, seed=100)],
        keyframe=[dict(win=0, feat_slot=B, n_cams=C)],
        stereo=[dict(win=0, pose=B, feat_slot=B, cam_a=0, cam_b=1)])


def run(full, w0, first_seen, world, reps):
    K, L, C = len(w0.poses), len(w0.landmarks), len(w0.cameras)
    F = K + 1
    ctxs = [capi.Context(0, 1) for _ in range(world)]
    pool = ThreadPoolExecutor(world)
    try:
        if world > 1:
            capi.Context.shard_connect_local(ctxs, max_frames=K, max_landmarks=L)
        s = Slide(list(enumerate(ctxs)), world, full, w0, first_seen, features=(F, C, N_KP, DESC))
        load(s, full, w0, F)
        J = jobs(w0, F)
        method = dict(detect="detect_describe_store_batch", track="track_3d2d_batch", match2d2d="match2d2d_batch",
                      ransac="ransac_3d2d_batch", keyframe="keyframe_overlap_batch", stereo="stereo_init_batch")
        kw = dict(detect=dict(uniformity_radius=40.0, max_keypoints=N_KP, desc_bytes=DESC))

        def call(name):
            fs = [pool.submit(lambda c=c: getattr(c, method[name])(J[name], **kw.get(name, {}))) for c in ctxs]
            return [f.result() for f in fs]

        rows = []
        for _ in range(reps + 1):
            row = {}
            t_frame = time.perf_counter()
            for name in CALLS:
                t0 = time.perf_counter()
                out = call(name)
                row[name + "_ms"] = 1e3 * (time.perf_counter() - t0)
                if name == "track":
                    row["associations"] = int(len(out[0][0]["assoc"]))
            row["frame_ms"] = 1e3 * (time.perf_counter() - t_frame)
            rows.append(row)
        timed = rows[1:]
        med = {k: float(np.median([r[k] for r in timed])) for k in [c + "_ms" for c in CALLS] + ["frame_ms"]}
        return dict(world=world, landmarks=L, reps=reps, median=med, associations=rows[0]["associations"])
    finally:
        pool.shutdown()
        for c in ctxs:
            c.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--landmarks", type=int, default=8000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--worlds", default="1,2,4")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    full, w0, first_seen = slide_problem(a.landmarks, extra=1)
    res = dict(card=card(), devices="one device; sharded ranks share it (exchange + redundant work, not multi-GPU scaling)",
               multi_gpu="not measured", runs=[run(full, w0, first_seen, int(w), a.reps) for w in a.worlds.split(",")])
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
