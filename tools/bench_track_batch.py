"""3D-2D tracking of the new frame against resident windows: okb_track_3d2d_batch against the per-round path, one JSON line.

For 1 / 132 / 528 cfg-2-shaped sessions (10 frames, stereo, 2 000 landmarks, about 400 keypoints per image, 48-byte
descriptors; eight seeded scenes of tests/track_scene.py dealt round-robin over the slots), each session tracks its
newest frame against its last three keyframes in both cameras (6 rounds, matchToKeyframes' 3D-2D loop):
  batch:  one okb_track_3d2d_batch over all sessions (pending edits committed inside; B's keypoints are re-set, untimed,
          before every repetition so that every repetition tracks a fresh frame);
  rounds: today's device part of the same work: okb_window_download_batch of every window's landmarks (the host's
          doSetup reads them), then one okb_hamming_match_batch per round over all sessions, with both descriptor lists
          and the gate arrays of every session uploaded again.  The host's doSetup / setBestMatch are not timed (they
          come on top), so this is a lower bound of the per-round path.
Host clock around work that ends in a device synchronise; the two alternate in the same run, best of --reps.  H2D / D2H
bytes per frame are computed from the shapes.  The card's name, power limit and max SM clock are read in the same run.

    python tools/bench_track_batch.py [--sizes 1,132,528] [--reps 5] [--out track_batch.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from okvis_b200 import abi, capi  # noqa: E402
import track_reference as tr  # noqa: E402
from track_scene import load, make_track_scene  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,132,528")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    sizes = [int(x) for x in a.sizes.split(",")]
    scenes = [make_track_scene(i, n_kp=400, n_frames=10, n_landmarks=2000, distortion=abi.DIST_RADTAN) for i in range(8)]
    D = 48
    # per scene, the arrays the host's doSetup makes for each round (for the per-round path's gate uploads)
    setups = []
    for sc in scenes:
        st = tr.TrackState(sc["window"], sc["store"], sc["lm_init"])
        setups.append([tr.setup_round(st, sc["pose_b"], sc["sb_b"], sc["feat_b"], *r) for r in sc["rounds"]["keyframes"]])
    result = dict(card=card(), workload="cfg-2-shaped sessions, 6 rounds (3 keyframes x 2 cameras), 48-byte descriptors",
                  note="rounds = download + one okb_hamming_match_batch per round; host doSetup / setBestMatch not timed", sizes={})
    for n in sizes:
        ctx = capi.Context(0, n)
        for s in range(n):
            load(ctx, s, scenes[s % 8])
        jobs = [dict(win=s, pose_b=scenes[s % 8]["pose_b"], sb_b=scenes[s % 8]["sb_b"], feat_slot_b=scenes[s % 8]["feat_b"],
                     rounds=scenes[s % 8]["rounds"]["keyframes"]) for s in range(n)]

        def reset_b():
            for s in range(n):
                sc = scenes[s % 8]
                for c in range(2):
                    e = sc["store"][(sc["feat_b"], c)]
                    ctx.set_features(s, sc["feat_b"], c, np.stack([e["kp"][:, 0], e["kp"][:, 1], e["size"]], 1), e["desc"], e["lm"], e["observed"])
            ctx.commit(0, n)

        round_jobs = []
        for r in range(6):
            js = []
            for s in range(n):
                sc, su = scenes[s % 8], setups[s % 8][r]
                fa, ca, cb = sc["rounds"]["keyframes"][r]
                A, B = sc["store"][(fa, ca)], sc["store"][(sc["feat_b"], cb)]
                g = abi.make_match_gate(abi.GATE_3D2D, B["kp"], B["size"], proj_into_b=su["proj"], proj_uncertainty=su["unc"])
                js.append(ctx.make_match_job(A["desc"], B["desc"], su["skipA"], su["skipB"], threshold=60.0, num_best=4, gate=g, want_topk=False))
            round_jobs.append(js)
        lms = [np.zeros((len(scenes[s % 8]["window"].landmarks), 4)) for s in range(n)]
        lm_ptrs = (C.POINTER(C.c_double) * n)(*[x.ctypes.data_as(C.POINTER(C.c_double)) for x in lms])

        def per_round():
            rc = capi.lib().okb_window_download_batch(ctx._h, 0, n, None, None, lm_ptrs, None)
            if rc != 0:
                raise capi.OkbError(rc, "okb_window_download_batch")
            for js in round_jobs:
                ctx.hamming_match_batch(js, D)

        best_b, best_r = float("inf"), float("inf")
        reset_b(); ctx.track_3d2d_batch(jobs); per_round()           # warm-up: buffers grown, modules loaded
        for _ in range(a.reps):
            reset_b()
            t0 = time.perf_counter(); out = ctx.track_3d2d_batch(jobs); best_b = min(best_b, time.perf_counter() - t0)
            t0 = time.perf_counter(); per_round(); best_r = min(best_r, time.perf_counter() - t0)
        # bytes per frame from the shapes
        nA = [[len(scenes[s % 8]["store"][r[:2]]["lm"]) for r in scenes[s % 8]["rounds"]["keyframes"]] for s in range(n)]
        nB = [[len(scenes[s % 8]["store"][(scenes[s % 8]["feat_b"], r[2])]["lm"]) for r in scenes[s % 8]["rounds"]["keyframes"]] for s in range(n)]
        # job table: 64 B per job, a 488-byte matcher entry (gate included) + 16 B round entry per (job, round)
        batch_h2d = n * 64 + sum(len(x) for x in nA) * (488 + 16)
        batch_d2h = sum(4 * (2 * 6 + 2) + 8 * sum(b) + 4 * sum(x) for x, b in zip(nA, nB))
        rounds_h2d = sum(sum(x) * (D + 1 + 16 + 32) + sum(b) * (D + 1 + 16 + 8) for x, b in zip(nA, nB))
        rounds_d2h = sum(32 * len(lms[s]) for s in range(n)) + sum(8 * sum(b) for b in nB)
        result["sizes"][str(n)] = dict(batch_ms=1e3 * best_b, rounds_device_ms=1e3 * best_r, speedup=best_r / best_b,
                                       matches=int(sum(int(o["num_matches"].sum()) for o in out)),
                                       batch_h2d_bytes=int(batch_h2d), batch_d2h_bytes=int(batch_d2h),
                                       rounds_h2d_bytes=int(rounds_h2d), rounds_d2h_bytes=int(rounds_d2h))
        ctx.close()
        print(json.dumps(result["sizes"][str(n)]), file=sys.stderr)
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
