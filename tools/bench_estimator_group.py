"""Host wall time per frame of N okvis::Estimator sessions through the C++ mirror, as JSON lines.

For each N, tests/shim/group_test.bin --bench N F runs F frames of the ThreadedKFVio cycle (addStates ->
addLandmark / addObservation -> optimize(10) -> applyMarginalizationStrategy(5, 3)) on N sessions of the scene of
shim_test.cpp --sliding, three ways:
  standalone_loop:     N standalone Estimators (one context each), called one after another;
  group_one_per_call:  one EstimatorGroup, every group call listing one session;
  group_batched:       one EstimatorGroup, every group call listing all N sessions.
The first 8 frames (first uploads, graph capture, the window filling up) are not timed.  Per timed frame it reports the
wall time of addStates + optimize + applyMarginalizationStrategy over all sessions, split into the time inside the
C-ABI calls that run and wait for device work (device_calls_ms) and the rest (host_bookkeeping_ms); the frontend's
addLandmark / addObservation calls are reported apart (observations_ms).  The standalone arm runs for N up to
--standalone-max only (one context per session).

    python tools/bench_estimator_group.py [--sessions 8 64 132 528] [--frames 16] [--standalone-max 132] [--out f.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
BIN = os.path.join(ROOT, "tests", "shim", "group_test.bin")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", type=int, nargs="+", default=[8, 64, 132, 528])
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--standalone-max", type=int, default=132)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not os.path.exists(BIN):
        raise SystemExit("%s not built: run __graft_entry__.build()" % BIN)
    lines = []
    for n in args.sessions:
        out = subprocess.run([BIN, "--bench", str(n), str(args.frames), str(args.standalone_max)], capture_output=True, text=True)
        if out.returncode != 0:
            raise SystemExit("group_test.bin --bench %d failed: %s%s" % (n, out.stdout, out.stderr))
        r = json.loads(out.stdout.strip().splitlines()[-1])
        r["card"] = card()          # name, power limit, max SM clock, SM clock, read right after the run
        lines.append(r)
        print(json.dumps(r), flush=True)
        for arm in ("standalone_loop", "group_one_per_call", "group_batched"):
            a = r[arm]
            if a is None:
                print("  N=%-4d %-19s not run (more than --standalone-max contexts)" % (n, arm), file=sys.stderr)
                continue
            print("  N=%-4d %-19s %9.2f ms/frame  (device calls %8.2f, host %8.2f; addStates %7.2f, optimize %8.2f, "
                  "marginalise %8.2f)" % (n, arm, a["ms_per_frame"], a["device_calls_ms"], a["host_bookkeeping_ms"],
                                          a["add_states_ms"], a["optimize_ms"], a["marginalize_ms"]), file=sys.stderr)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in lines))


if __name__ == "__main__":
    main()
