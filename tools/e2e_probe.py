"""Where does the end-to-end (host buffers) time go?  Times upload / optimize / download of Be windows separately."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from okvis_b200 import capi, synthetic
Be = int(sys.argv[1]) if len(sys.argv) > 1 else 132
ctx = capi.Context(0, 2 * Be)
ws = [synthetic.make_window(2, i) for i in range(8)]
rw = [ws[i % 8] for i in range(Be)]
descs = ctx.make_descs(rw)
for b in (0, Be):
    ctx.upload_batch(b, rw, 8, descs)
outs = {b: ctx.alloc_outputs(b, Be) for b in (0, Be)}
ctx.optimize(0, Be, max_iterations=10)
torch.cuda.synchronize()
for T in (1, 2, 4, 8, 16):
    t0 = time.perf_counter(); ctx.upload_batch(0, rw, T, descs); t1 = time.perf_counter()
    torch.cuda.synchronize(); t2 = time.perf_counter()
    ctx.optimize(0, Be, max_iterations=10); t3 = time.perf_counter()
    ctx.download_batch(0, Be, outs[0]); t4 = time.perf_counter()
    print("threads %2d: upload host %.2f ms (+drain %.2f), optimize %.2f ms, download %.2f ms" % (
        T, (t1 - t0) * 1e3, (t2 - t1) * 1e3, (t3 - t2) * 1e3, (t4 - t3) * 1e3), flush=True)
for T in (2, 4, 8):
    def run(n):
        ctx.upload_batch(0, rw, T, descs); pending = None
        for st in range(n):
            base = (st % 2) * Be
            ctx.optimize_async(base, Be, max_iterations=10)
            if pending is not None: ctx.download_batch(pending, Be, outs[pending])
            if st + 1 < n: ctx.upload_batch(((st + 1) % 2) * Be, rw, T, descs)
            ctx.optimize_finish(base, Be)
            pending = base
        ctx.download_batch(pending, Be, outs[pending])
    run(2)
    t0 = time.perf_counter(); run(6); dt = time.perf_counter() - t0
    print("pipelined, %d threads: %.2f ms/step -> %.0f iter/s" % (T, dt / 6 * 1e3, 6 * Be * 10 / dt), flush=True)
# which leg fails to overlap?
T = 8
def loop(n, do_up, do_down):
    ctx.upload_batch(0, rw, T, descs); ctx.upload_batch(Be, rw, T, descs); pending = None
    t0 = time.perf_counter()
    tt = {"async": 0.0, "down": 0.0, "up": 0.0, "finish": 0.0}
    for st in range(n):
        base = (st % 2) * Be
        a = time.perf_counter(); ctx.optimize_async(base, Be, max_iterations=10); b = time.perf_counter()
        if do_down and pending is not None: ctx.download_batch(pending, Be, outs[pending])
        c = time.perf_counter()
        if do_up and st + 1 < n: ctx.upload_batch(((st + 1) % 2) * Be, rw, T, descs)
        d = time.perf_counter()
        ctx.optimize_finish(base, Be); e = time.perf_counter()
        tt["async"] += b - a; tt["down"] += c - b; tt["up"] += d - c; tt["finish"] += e - d
        pending = base
    dt = time.perf_counter() - t0
    return dt / n * 1e3, {k: round(v / n * 1e3, 2) for k, v in tt.items()}
for up, down in ((False, False), (False, True), (True, False), (True, True)):
    loop(2, up, down)
    print("upload=%d download=%d: %.2f ms/step  %s" % (up, down, *loop(6, up, down)), flush=True)
