"""Per-kernel device time of bench.py's resident workload, from torch.profiler (CUDA activities).

The workload is the one bench.py times: `--batch` resident cfg-2 windows (the same seeded synthetic windows), and
per step a device-side reset plus optimize(10), with the library's event profiling on as in bench.py's timed
region.  Only the profiled steps are traced.  The tracer slows the host, so take throughput from bench.py and only
shares from this table.

    python tools/kernel_table.py [--batch 528] [--steps 2] [--out DIR]

Prints a markdown table.  With --out it also writes DIR/kernel_table.json and DIR/kernel_table.md.
"""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ITERS = 10


def short_name(name):
    """'void okb::k_solve<512>(okb::WinDev const*, ...)' -> 'k_solve<512>'; copies and memsets keep their names."""
    if name.startswith(("Memcpy", "Memset")):
        return name
    m = re.search(r"([A-Za-z_][A-Za-z0-9_]*(?:<[^()]*>)?)\s*\(", name)
    return m.group(1) if m else name


def gpu_identity():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        name, power, sm_max = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit_w": float(power), "sm_max_mhz": float(sm_max)}
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=528, help="resident windows (bench.py's default)")
    ap.add_argument("--distinct", type=int, default=8, help="distinct synthetic windows, replicated to fill the batch")
    ap.add_argument("--steps", type=int, default=2, help="profiled steps")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", help="directory for kernel_table.json / kernel_table.md")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from okvis_b200 import capi, synthetic

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B = args.batch
    windows = [synthetic.make_window(2, i) for i in range(args.distinct)]
    ctx = capi.Context(0, B)
    try:
        ctx.upload_batch(0, [windows[i % len(windows)] for i in range(B)])
        ctx.profile_enable(True)

        def step():
            ctx.reset(0, B)
            return ctx.optimize(0, B, max_iterations=ITERS)

        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize(dev)
        launches0 = ctx.kernel_launches
        iters = 0
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                iters += sum(s["iterations"] for s in step())
            torch.cuda.synchronize(dev)
        launches = ctx.kernel_launches - launches0
    finally:
        ctx.close()

    totals = {}
    for e in prof.key_averages():
        us = getattr(e, "self_device_time_total", None)
        if us is None:
            us = e.self_cuda_time_total
        if us <= 0:
            continue
        k = short_name(e.key)
        t, n = totals.get(k, (0.0, 0))
        totals[k] = (t + us, n + e.count)
    all_us = sum(t for t, _ in totals.values())
    rows = sorted(({"kernel": k, "launches": n, "total_ms": t / 1e3, "mean_us": t / max(n, 1), "share": t / all_us}
                   for k, (t, n) in totals.items()), key=lambda r: -r["total_ms"])
    res = {"gpu": gpu_identity(), "batch": B, "steps": args.steps, "iterations": iters, "library_launches": launches,
           "device_ms_per_step": all_us / 1e3 / args.steps, "kernels": rows}

    g = res["gpu"] or {}
    md = ["%s, power limit %s W: %d resident cfg-2 windows, %d profiled steps of reset + optimize(%d), "
          "%.2f ms of device time per step, %d library launches per step" % (
              g.get("name", "unknown GPU"), g.get("power_limit_w", "?"), B, args.steps, ITERS, res["device_ms_per_step"],
              launches // args.steps), "",
          "| kernel | launches per step | ms per step | mean us | share |", "|---|---|---|---|---|"]
    for r in rows:
        md.append("| `%s` | %d | %.3f | %.1f | %.1f %% |" % (r["kernel"], r["launches"] // args.steps, r["total_ms"] / args.steps,
                                                           r["mean_us"], 100 * r["share"]))
    text = "\n".join(md)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "kernel_table.json"), "w") as f:
            json.dump(res, f, indent=1)
        with open(os.path.join(args.out, "kernel_table.md"), "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
