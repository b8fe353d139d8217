"""Where does the e2e leg lose time?  Variants of the streaming loop on 528-window ranges."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from okvis_b200 import capi, synthetic
B = int(sys.argv[1]) if len(sys.argv) > 1 else 528
ctx = capi.Context(0, 2 * B)
ws = [synthetic.make_window(2, i) for i in range(8)]
rw = [ws[i % 8] for i in range(B)]
descs = ctx.make_descs(rw)
for base in (0, B):
    for i, w in enumerate(rw):
        ctx.reserve(base + i, len(w.poses), len(w.landmarks), len(w.obs) + 4096, len(w.imu_samples) + 256)
    ctx.upload_batch(base, rw, 12, descs)
outs = {b: ctx.alloc_outputs(b, B) for b in (0, B)}
prep = {b: [ctx.prepare_readd_newest(b + i, w) for i, w in enumerate(rw)] for b in (0, B)}

def run(n, do_reset, do_readd, do_download, tag):
    host = dict(opt=0.0, down=0.0, reset=0.0, readd=0.0, commit=0.0, finish=0.0)
    def up(base):
        t = time.perf_counter()
        if do_reset: ctx.reset(base, B)
        host["reset"] += time.perf_counter() - t; t = time.perf_counter()
        if do_readd: ctx.readd_newest(prep[base])
        host["readd"] += time.perf_counter() - t; t = time.perf_counter()
        if do_readd: ctx.commit(base, B)
        host["commit"] += time.perf_counter() - t
    it = 0
    up(0)
    pending = None
    t0 = time.perf_counter()
    for st in range(n):
        base = (st % 2) * B
        t = time.perf_counter(); ctx.optimize_async(base, B, max_iterations=10); host["opt"] += time.perf_counter() - t
        if pending is not None and do_download:
            t = time.perf_counter(); ctx.download_batch(pending, B, outs[pending]); host["down"] += time.perf_counter() - t
        if st + 1 < n: up(((st + 1) % 2) * B)
        t = time.perf_counter(); ss = ctx.optimize_finish(base, B); host["finish"] += time.perf_counter() - t
        it += sum(x["iterations"] for x in ss)
        pending = base
    dt = time.perf_counter() - t0
    print("%-28s %.0f it/s  %.2f ms/step | host ms/step: %s" % (tag, it / dt, dt / n * 1e3, {k: round(v / n * 1e3, 2) for k, v in host.items()}))

for rep in range(2):
    run(6, False, False, False, "optimize only")
    run(6, True, False, False, "+ reset")
    run(6, True, False, True, "+ reset + download")
    run(6, True, True, False, "+ reset + readd/commit")
    run(6, True, True, True, "full")
