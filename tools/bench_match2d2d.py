"""2D-2D landmark initialisation against earlier frames (the 2D-2D rounds of matchToKeyframes / matchToLastFrame):
okb_match2d2d_batch, with okb_stereo_init_batch timed at the same shape in the same run, one JSON line.

For 1 / 132 / 528 cfg-2-shaped sessions (stereo, about 400 keypoints per image, 48-byte descriptors; four seeded scenes
of tests/temporal_scene.py dealt round-robin over the slots):
  call:       one okb_match2d2d_batch over all sessions, each matching its older frame's camera 0 against the current
              frame's camera 0 (with the current frame's speed/bias block);
  per frame:  the 3 C = 6 rounds a stereo session runs per frame (two keyframes and the last frame, each camera), one
              call per round as the mirror issues them.  The same two jobs are issued three times each and no records
              are applied between the calls: the time is the device work and call overhead only, without the host's
              setBestMatch bookkeeping that the mirror runs between rounds;
  stereo:     one okb_stereo_init_batch of the current frame's cameras 0 -> 1.
Host clock around work that ends in a device synchronise; the three alternate in the same run, best of --reps.  H2D /
D2H bytes per call are computed from the shapes: H2D up256(job table) + match table, D2H sum(16 + 56 nB).  The card's
name, power limit and max SM clock are read in the same run.

    python tools/bench_match2d2d.py [--sizes 1,132,528] [--reps 5] [--out match2d2d.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time


ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from okvis_b200 import abi, capi  # noqa: E402
from oracle import oracle_py  # noqa: E402
from temporal_scene import jobs, load, make_temporal_scene, stereo_jobs  # noqa: E402

# device table entries of the call (okb_frontend.cu): StereoJobDev 72 B, MatchJobDev with its 2D-2D gate 488 B
JOB_BYTES, MATCH_BYTES, RECORD_BYTES = 72, 488, 56


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def up256(v):
    return (v + 255) & ~255


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,132,528")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    sizes = [int(x) for x in a.sizes.split(",")]
    D = 48
    scenes = [make_temporal_scene(i, abi.DIST_RADTAN, n_kp=400, desc_bytes=D, oracle=oracle_py) for i in range(4)]
    result = dict(card=card(), desc_bytes=D, sizes={})
    for n in sizes:
        ctx = capi.Context(0, n)
        for s in range(n):
            load(ctx, s, scenes[s % 4])
        rounds = [[dict(jobs(scenes[s % 4])[c], win=s) for s in range(n)] for c in (0, 1)]
        sjobs = [dict(stereo_jobs(scenes[s % 4])[0], win=s) for s in range(n)]
        ctx.match2d2d_batch(rounds[0]); ctx.match2d2d_batch(rounds[1]); ctx.stereo_init_batch(sjobs)
        t_call, t_frame, t_stereo = [], [], []
        for _ in range(a.reps):
            t0 = time.perf_counter(); ctx.match2d2d_batch(rounds[0]); t_call.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            for r in range(6):
                ctx.match2d2d_batch(rounds[r % 2])
            t_frame.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); ctx.stereo_init_batch(sjobs); t_stereo.append(time.perf_counter() - t0)
        nB = [len(scenes[s % 4]["state"]["store"][(scenes[s % 4]["frames"]["feat_slot_b"], 0)]["lm"]) for s in range(n)]
        h2d = up256(up256(JOB_BYTES * n) + MATCH_BYTES * n)
        d2h = sum(16 + RECORD_BYTES * b for b in nB)
        result["sizes"][n] = dict(call_ms=1e3 * min(t_call), frame_6_rounds_ms=1e3 * min(t_frame), stereo_call_ms=1e3 * min(t_stereo),
                                  h2d_bytes_per_call=h2d, d2h_bytes_per_call=d2h)
        ctx.close()
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
