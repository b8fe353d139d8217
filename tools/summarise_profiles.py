"""Turns the ncu outputs gathered by tools/collect_profiles.sh (gpurun_out/) into the tracked summaries under
profiles/: per-kernel share of the step from the launch list, DRAM traffic and pipe utilisation of each
solver kernel from its --set full capture."""
import csv, json, os, shutil, sys
from collections import defaultdict
R = sys.argv[1] if len(sys.argv) > 1 else "r01"
B = int(sys.argv[2]) if len(sys.argv) > 2 else 528
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G, P = os.path.join(ROOT, "gpurun_out"), os.path.join(ROOT, "profiles")

def read_csv(path):
    rows = [r for r in csv.reader(open(path)) if r and not r[0].startswith("==")]
    if not rows:
        return [], []
    return rows[0], rows[1:]

# ---- launch list
hdr, rows = read_csv(os.path.join(G, f"{R}_launches_bench.csv"))
ix = {h: i for i, h in enumerate(hdr)}
tot = defaultdict(float); cnt = defaultdict(int)
for r in rows:
    if r[ix["Metric Name"]] != "gpu__time_duration.sum":
        continue
    name = r[ix["Kernel Name"]].split("(")[0].replace("okb::", "").replace("void ", "")
    v = float(r[ix["Metric Value"]].replace(",", ""))
    unit = r[ix["Metric Unit"]]
    v *= {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}.get(unit, 1.0)
    tot[name] += v; cnt[name] += 1
total = sum(tot.values())
shutil.copy(os.path.join(G, f"{R}_launches_bench.csv"), os.path.join(P, f"{R}_launches_bench.csv"))

# ---- per-kernel full captures
kern = {}
for k in ("k_landmarks", "k_schur", "k_solve", "k_imu", "k_quality"):
    raw = os.path.join(G, f"{R}_{k}_raw.csv")
    det = os.path.join(G, f"{R}_{k}_details.csv")
    if not os.path.exists(raw):
        continue
    h, rr = read_csv(raw)
    if not rr:
        continue
    vals = dict(zip(h, rr[-1]))
    def f(key):
        for kk, v in vals.items():
            if kk.startswith(key):
                try: return float(v.replace(",", ""))
                except ValueError: return None
        return None
    units = dict(zip(h, rr[0])) if len(rr) > 1 else {}
    def with_unit(key, target):
        v = f(key)
        if v is None: return None
        u = next((units[kk] for kk in units if kk.startswith(key)), "")
        scale = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1e-3, "us": 1, "ms": 1e3}.get(u, 1)
        return v * scale
    kern[k] = dict(duration_us=with_unit("gpu__time_duration.sum", "us"), dram_read_bytes=with_unit("dram__bytes_read.sum", "byte"),
                   dram_write_bytes=with_unit("dram__bytes_write.sum", "byte"), warp_inst=f("smsp__inst_executed.sum"),
                   fp64_pipe_pct=f("sm__inst_executed_pipe_fp64"), warps_active_pct=f("sm__warps_active"))
    if os.path.exists(det):
        shutil.copy(det, os.path.join(P, f"{R}_{k}_details.csv"))
json.dump({"windows": B, "note": "one ncu --set full capture per kernel, tools/prof_small.py %d 4 (cfg-2 windows), per launch" % B,
           "kernels": kern}, open(os.path.join(P, f"{R}_traffic.json"), "w"), indent=1)

with open(os.path.join(P, f"{R}_summary.md"), "w") as f_:
    f_.write(f"# {R}: ncu summary of the solver kernels (H100, cfg-2 windows)\n\n")
    f_.write(f"## Launch list of `bench.py --steps 2 --warmup 3` (first 700 launches; `{R}_launches_bench.csv`)\n\n")
    f_.write("per-launch times under ncu are cold-cache and serialised: read the SHARE, not the absolute\n\n")
    f_.write("| kernel | launches | total us | mean us | share |\n|---|---|---|---|---|\n")
    for k, v in sorted(tot.items(), key=lambda x: -x[1]):
        f_.write(f"| {k} | {cnt[k]} | {v:.0f} | {v / cnt[k]:.1f} | {100 * v / total:.1f} % |\n")
    f_.write(f"\n## `--set full` captures at {B} resident windows (`{R}_<kernel>_details.csv`, `{R}_traffic.json`)\n\n")
    f_.write("| kernel | duration us | DRAM read MB | DRAM write MB | warp instr (M) | FP64 pipe % | warps active % |\n|---|---|---|---|---|---|---|\n")
    for k, v in kern.items():
        g = lambda x, s=1.0: "n/a" if v[x] is None else f"{v[x] / s:.1f}"
        f_.write(f"| {k} | {g('duration_us')} | {g('dram_read_bytes', 1e6)} | {g('dram_write_bytes', 1e6)} | {g('warp_inst', 1e6)} | {g('fp64_pipe_pct')} | {g('warps_active_pct')} |\n")
    # frontend / marginalisation captures and the sanitizer logs travel as they are
    fl = os.path.join(G, f"{R}_launches_frontend.csv")
    if os.path.exists(fl):
        shutil.copy(fl, os.path.join(P, f"{R}_launches_frontend.csv"))
        h2, r2 = read_csv(fl)
        i2 = {h: i for i, h in enumerate(h2)}
        f_.write("\n## Frontend kernels (`tools/prof_frontend.py`: cfg-3 image, production image, 1000 x 1000 match, candidate lists; second repetition)\n\n")
        f_.write("| kernel | grid | block | us |\n|---|---|---|---|\n")
        for r in r2[len(r2) // 2:]:
            v = float(r[i2["Metric Value"]].replace(",", "")) * {"ns": 1e-3, "us": 1.0, "ms": 1e3}.get(r[i2["Metric Unit"]], 1.0)
            f_.write(f"| {r[i2['Kernel Name']].split('(')[0].replace('void ', '').replace('<unnamed>::', '')} | {r[i2['Grid Size']]} | {r[i2['Block Size']]} | {v:.1f} |\n")
    for k in ("k_uniformity", "k_hamming_topk", "k_harris", "k_describe", "k_marginalize"):
        det = os.path.join(G, f"{R}_{k}_details.csv")
        if os.path.exists(det) and os.path.getsize(det) > 0:
            shutil.copy(det, os.path.join(P, f"{R}_{k}_details.csv"))
    f_.write("\n## compute-sanitizer (`tools/sanitize_run.py`: cfg-1 / reduced cfg-2 / cfg-5 optimize, 2-rank sharded solve, resident edits, marginalisation, frontend)\n\n")
    for tool in ("memcheck", "racecheck", "synccheck"):
        sp = os.path.join(G, f"{R}_sanitizer_{tool}.txt")
        if os.path.exists(sp):
            shutil.copy(sp, os.path.join(P, f"{R}_sanitizer_{tool}.txt"))
            tail = [l.strip() for l in open(sp) if "ERROR SUMMARY" in l or "RACECHECK SUMMARY" in l]
            f_.write(f"* {tool}: {tail[-1] if tail else 'see log'}\n")
print(open(os.path.join(P, f"{R}_summary.md")).read())
