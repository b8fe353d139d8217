"""Times okb_keyframe_overlap_batch at 1 / 132 / 528 sessions shaped like cfg 2 (two cameras, 400 keypoints each)
against a host loop over the same images: cv2 (convexHull, contourArea, pointPolygonTest, as the reference calls them)
when this machine's Python has it, else the NumPy restatement tests/keyframe_reference.py -- the output says which.
Device times are a host clock around the call, which returns after its H2D copy, launch and D2H copy have synchronised; host times a
perf_counter around the loop.  Prints the card name and power limit from the same run, and one JSON line."""
import argparse
import ctypes as C
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
import keyframe_reference as ref  # noqa: E402
import keyframe_scene as S  # noqa: E402


def host_decision_cv2(cv2, images):
    overlap = ratio = 0.0
    for kp, lm in images:
        pts = kp.astype(np.float32)
        m = pts[lm >= 0]
        if len(pts) < 3:
            continue
        hull = cv2.convexHull(pts)
        if len(m) < 3:
            continue
        mh = cv2.convexHull(m)
        a, am = cv2.contourArea(hull), cv2.contourArea(mh)
        inside = 0
        if len(mh) > 2:
            for p in pts:
                if cv2.pointPolygonTest(mh, (float(p[0]), float(p[1])), False) > 0:
                    inside += 1
        o = am / a if a else float("nan")
        r = len(m) / inside if inside else float("inf")
        overlap, ratio = ref.std_max(o, overlap), ref.std_max(r, ratio)
    return not (overlap > np.float32(0.6) and ratio > np.float32(0.2))


def host_decision_numpy(images):
    return S.session_values(images)["need_keyframe"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", default="1,132,528")
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("card:", q)
    try:
        import cv2
        host_name = "cv2 %s" % cv2.__version__
    except ImportError:
        cv2 = None
        host_name = "numpy restatement (cv2 not installed)"
    print("host loop:", host_name)
    rng = np.random.default_rng(2024)
    pool = [[S.random_image(rng) for _ in range(2)] for _ in range(16)]
    rows = []
    for n in [int(x) for x in args.sessions.split(",")]:
        ctx = capi.Context(0, n)
        for s in range(n):
            S.load(ctx, s, pool[s % len(pool)])
        jobs = [dict(win=s, feat_slot=1, n_cams=2) for s in range(n)]
        got = ctx.keyframe_overlap_batch(jobs)          # warm-up (module load, buffers)
        for s in range(min(n, 16)):
            assert got[s]["need_keyframe"] == S.session_values(pool[s % len(pool)])["need_keyframe"]
        # the C call alone: the job table and its outputs are built once, outside the timed loop
        arr = (abi.KeyframeJob * n)()
        cams = (abi.KeyframeCam * (2 * n))()
        outs = (abi.KeyframeResult * n)()
        for s in range(n):
            arr[s].win, arr[s].feat_slot, arr[s].n_cams = s, 1, 2
            arr[s].overlap_threshold, arr[s].matching_ratio_threshold = 0.6, 0.2
            arr[s].cams = C.cast(C.byref(cams, 2 * s * C.sizeof(abi.KeyframeCam)), C.POINTER(abi.KeyframeCam))
            arr[s].out = C.cast(C.byref(outs, s * C.sizeof(abi.KeyframeResult)), C.POINTER(abi.KeyframeResult))
        ts = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            rc = capi.lib().okb_keyframe_overlap_batch(ctx._h, n, arr)
            ts.append(time.perf_counter() - t0)
            assert rc == 0
        assert [bool(outs[s].need_keyframe) for s in range(n)] == [g["need_keyframe"] for g in got]
        dev_ms = 1e3 * float(np.median(ts))
        host_n = min(n, 132)
        t0 = time.perf_counter()
        for s in range(host_n):
            if cv2 is not None:
                host_decision_cv2(cv2, pool[s % len(pool)])
            else:
                host_decision_numpy(pool[s % len(pool)])
        host_ms = 1e3 * (time.perf_counter() - t0) * n / host_n
        rows.append(dict(sessions=n, device_call_ms=round(dev_ms, 4), host_loop_ms=round(host_ms, 3)))
        print("sessions %4d  device call %.3f ms (median of %d, host clock around the synchronising call)  host loop %.2f ms"
              % (n, dev_ms, args.reps, host_ms))
        ctx.close()
    print(json.dumps(dict(card=q, host_loop=host_name, rows=rows)))


if __name__ == "__main__":
    main()
