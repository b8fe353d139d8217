"""Timing probe: B=1 latency, batch throughput, per-kernel and per-phase split."""
import os, sys, time, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from okvis_b200 import capi, synthetic
out = open(os.path.join(ROOT, "gpurun_out", "perf_probe.txt"), "w")
def P(*a):
    s = " ".join(str(x) for x in a); print(s); out.write(s + "\n"); out.flush()
ws = [synthetic.make_window(2, i) for i in range(4)]
for B in (1, 132, 528):
    ctx = capi.Context(0, B)
    for i in range(B):
        ctx.upload(i, ws[i % 4])
    ctx.optimize(0, B, max_iterations=10)
    for rep in range(2):
        ctx.reset(0, B)
        ctx.profile_enable(True)
        t = time.time(); s = ctx.optimize(0, B, max_iterations=10); dt = time.time() - t
        pr = ctx.profile_read()
        its = sum(x["iterations"] for x in s)
        P("B=%d wall %.4f s  %.0f iter/s  device %.5f s | A %.3f ms/launch x%d, S %.3f ms/launch x%d, Q %.3f ms" % (
            B, dt, its / dt, s[0]["solve_time_s"], pr["landmarks_ms"] / max(pr["landmarks_launches"], 1), pr["landmarks_launches"],
            pr["solve_ms"] / max(pr["solve_launches"], 1), pr["solve_launches"], pr["quality_ms"]))
        P("   phases(us, summed over rounds):", json.dumps({k: round(v, 1) for k, v in ctx.debug_phase_us(0).items()}))
    ctx.close()
