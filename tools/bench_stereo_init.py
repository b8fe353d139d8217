"""Stereo landmark initialisation (matchStereo's 2D-2D match): okb_stereo_init_batch against today's device part, one
JSON line.

For 1 / 132 / 528 cfg-2-shaped sessions (stereo, 400 keypoints per image, 48-byte descriptors; four seeded scenes of
tests/stereo_scene.py dealt round-robin over the slots), each session matches its newest frame's camera 0 against
camera 1:
  call:   one okb_stereo_init_batch over all sessions (the device backProjects, matches, triangulates and decides
          canBeInitialized; records come back);
  today:  one okb_hamming_match_batch with a 2D-2D gate, one job per session, with both descriptor lists and the
          host-built bearings and ray sigmas uploaded.  The host's backProject, doSetup and setBestMatch
          (stereoTriangulate, getUncertainty) are not timed: they come on top, so this is a lower bound.
Host clock around work that ends in a device synchronise; the two alternate in the same run, best of --reps.  H2D / D2H
bytes per frame are computed from the shapes.  The card's name, power limit and max SM clock are read in the same run.

    python tools/bench_stereo_init.py [--sizes 1,132,528] [--reps 5] [--out stereo_init.json]
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
import stereo_init_reference as ref  # noqa: E402
from stereo_scene import load, make_stereo_scene  # noqa: E402

# device table entries of the call (okb_frontend.cu): StereoJobDev 64 B, MatchJobDev with its 2D-2D gate 488 B
JOB_BYTES, MATCH_BYTES, RECORD_BYTES = 64, 488, 56


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
    scenes = [make_stereo_scene(i, abi.DIST_RADTAN, n_kp=400, desc_bytes=D, oracle=oracle_py) for i in range(4)]
    gates = []
    for sc in scenes:
        g = ref.setup(sc["state"], sc["job"])
        A, B = sc["state"]["store"][(sc["job"]["feat_slot"], 0)], sc["state"]["store"][(sc["job"]["feat_slot"], 1)]
        gates.append((A, B, g, ref.gate_struct(g)))
    result = dict(card=card(), desc_bytes=D, sizes={})
    for n in sizes:
        ctx = capi.Context(0, n)
        for s in range(n):
            load(ctx, s, scenes[s % 4])
        jobs = [dict(scenes[s % 4]["job"], win=s) for s in range(n)]
        mjobs = []
        for s in range(n):
            A, B, g, gate = gates[s % 4]
            mjobs.append(ctx.make_match_job(A["desc"], B["desc"], skipA=g["skipA"], skipB=g["skipB"], threshold=60.0, num_best=4, gate=gate, want_topk=False))
        ctx.stereo_init_batch(jobs)
        ctx.hamming_match_batch(mjobs, D)
        t_call, t_today = [], []
        for _ in range(a.reps):
            t0 = time.perf_counter(); ctx.stereo_init_batch(jobs); t_call.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); ctx.hamming_match_batch(mjobs, D); t_today.append(time.perf_counter() - t0)
        nA = [len(gates[s % 4][0]["lm"]) for s in range(n)]
        nB = [len(gates[s % 4][1]["lm"]) for s in range(n)]
        call_h2d = up256(JOB_BYTES * n) + up256(MATCH_BYTES * n)
        call_d2h = sum(16 + RECORD_BYTES * b for b in nB)
        today_h2d = MATCH_BYTES * n + sum((x + y) * D + x + y + 8 * (2 * y + y + 2 * x + x + 3 * x + 3 * y + x + y) for x, y in zip(nA, nB))
        today_d2h = sum(8 * y for y in nB)
        result["sizes"][n] = dict(call_ms=1e3 * min(t_call), today_device_ms=1e3 * min(t_today), call_h2d_bytes=call_h2d,
                                  call_d2h_bytes=call_d2h, today_h2d_bytes=today_h2d, today_d2h_bytes=today_d2h)
        ctx.close()
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
