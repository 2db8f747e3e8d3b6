#!/usr/bin/env python3
"""gpurun_out/launches_<tag>.csv (tools/profile3.sh: per launch gpu__time_duration, dram bytes read / written) ->
profiles/<round>_launches_<tag>.{csv,md} and profiles/dominant_kernel_traffic.json (DRAM bytes per image of every
pipeline stage, the figure bench.py reports as roofline.traffic);  gpurun_out/prof_<tag>_<kernel>.ncu-rep ->
profiles/<round>_<tag>_<kernel>.txt.      usage: profile_digest3.py <tag> [round] [images]"""
import csv, json, os, re, shutil, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
tag = sys.argv[1]; rnd = sys.argv[2] if len(sys.argv) > 2 else "r02"; nimg = int(sys.argv[3]) if len(sys.argv) > 3 else 16
src = os.path.join(ROOT, "gpurun_out", f"launches_{tag}.csv")
rows = [r for r in csv.reader(open(src)) if r and r[0].isdigit()]
# kernel -> pipeline stage (the names b200jpeg_last_stage_times reports)
STAGE = [("k_forward", "forward"), ("k_prep_planes", "smooth_planes"), ("k_import_coefs", "forward"), ("k_dummy", "dummy"), ("k_gather_comp", "trellis_stats"),
         ("k_sort", "trellis_ac"), ("k_trellis_ac", "trellis_ac"), ("k_trellis_eob", "trellis_ac"), ("k_qopt", "trellis_ac"), ("k_trellis_dc", "trellis_dc"), ("k_dc_collect", "trellis_dc"),
         ("k_gather_seq", "scan_stats"), ("k_gather_prog", "scan_stats"), ("k_seed_hist", "scan_stats"), ("k_gen_tables", "tables"), ("k_block_bits", "block_bits"),
         ("k_scan_layout", "scan_layout"), ("k_zero_stream", "encode"), ("k_encode", "encode"), ("k_stuff", "stuff"), ("k_prog", "eobrun_runs"), ("k_select_al", "select_al")]
def stage_of(name):
    for pre, st in STAGE:
        if name.startswith(pre): return st
    return "other"
launch = {}            # id -> dict
for r in rows:
    d = launch.setdefault(r[0], {"name": re.sub(r"\(.*", "", r[4]).replace("void ", "").replace("b200::", ""), "grid": r[8], "block": r[7]})
    val = float(r[14]); unit = r[13]
    if r[12].startswith("gpu__time"): d["ns"] = val * {"ns": 1, "us": 1e3, "ms": 1e6}.get(unit, 1)
    else:
        mult = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1)
        d["rd" if "read" in r[12] else "wr"] = val * mult
per = {}
for d in launch.values():
    p = per.setdefault(d["name"], {"n": 0, "ns": 0.0, "rd": 0.0, "wr": 0.0, "grid": d["grid"], "block": d["block"]})
    p["n"] += 1; p["ns"] += d.get("ns", 0); p["rd"] += d.get("rd", 0); p["wr"] += d.get("wr", 0); p["grid"] = d["grid"]
tot = sum(p["ns"] for p in per.values())
stages = {}
for name, p in per.items():
    s = stages.setdefault(stage_of(name), {"ns": 0.0, "bytes": 0.0}); s["ns"] += p["ns"]; s["bytes"] += p["rd"] + p["wr"]
# the bench step runs W warm-up + K timed + one single-stream pass: every kernel appears (launches / images-per-chunk) times
passes = max(1, min(p["n"] for n_, p in per.items() if n_.startswith("k_forward")) if any(n_.startswith("k_forward") for n_ in per) else 1)
os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)      # git-ignored output directory
out = os.path.join(ROOT, "profiles", f"{rnd}_launches_{tag}.md")
with open(out, "w") as f:
    f.write(f"# ncu launch list `{tag}` (`tools/profile3.sh {tag}`: bench.py --batch {nimg} --steps 1 --warmup 1, every launch, "
            "`--metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none`)\n\n")
    f.write(f"Per-launch times under ncu are cold-cache and serialised: compare SHARES with `roofline.stage_ms`, not absolutes.  {passes} passes over {nimg} images of 3840x2160.\n\n")
    f.write("| kernel | launches | total us | share | DRAM read MB | DRAM written MB | grid (last) | block |\n|---|---|---|---|---|---|---|---|\n")
    for name in sorted(per, key=lambda k: -per[k]["ns"]):
        p = per[name]
        f.write(f"| `{name}` | {p['n']} | {p['ns'] / 1e3:.1f} | {p['ns'] / tot * 100:.1f} % | {p['rd'] / 1e6:.1f} | {p['wr'] / 1e6:.1f} | {p['grid']} | {p['block']} |\n")
    f.write(f"\nTotal device time in kernels: {tot / 1e6:.3f} ms over {len(launch)} launches.\n\n")
    f.write("| stage | share of kernel time | DRAM MB per image |\n|---|---|---|\n")
    for st in sorted(stages, key=lambda k: -stages[k]["ns"]):
        f.write(f"| {st} | {stages[st]['ns'] / tot * 100:.1f} % | {stages[st]['bytes'] / passes / nimg / 1e6:.1f} |\n")
    f.write(f"\nSum over stages: {sum(s['bytes'] for s in stages.values()) / passes / nimg / 1e6:.1f} MB of DRAM traffic per image.\n")
print(open(out).read())
shutil.copy(src, os.path.join(ROOT, "profiles", f"{rnd}_launches_{tag}.csv"))
dom = max(stages, key=lambda k: stages[k]["ns"])
json.dump({"kernel": dom, "dram_bytes_per_image": stages[dom]["bytes"] / passes / nimg,
           "per_stage_dram_bytes_per_image": {k: v["bytes"] / passes / nimg for k, v in stages.items()},
           "source": f"profiles/{rnd}_launches_{tag}.csv: ncu dram__bytes_read.sum + dram__bytes_write.sum of every launch of the stage, {nimg} images of 3840x2160 "
                     f"(tools/profile3.sh + tools/profile_digest3.py; generated, not hand-edited)"},
          open(os.path.join(ROOT, "profiles", "dominant_kernel_traffic.json"), "w"), indent=1)
for fn in sorted(os.listdir(os.path.join(ROOT, "gpurun_out"))):
    m = re.match(rf"prof_{tag}_(.+)\.ncu-rep$", fn)
    if not m: continue
    k = m.group(1)
    txt = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ncu_summary.py"), os.path.join(ROOT, "gpurun_out", fn)], capture_output=True, text=True).stdout
    st = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ncu_stalls.py"), os.path.join(ROOT, "gpurun_out", fn), "6"], capture_output=True, text=True).stdout
    with open(os.path.join(ROOT, "profiles", f"{rnd}_{tag}_{k}.txt"), "w") as f:
        f.write(f"# ncu --set full --clock-control none --import-source on, kernel {k}, capture {tag} (batch {nimg} of 3840x2160, one launch)\n"
                "# headline metrics, hot SASS regions (instruction index range, #instr, executions per instr, share of warp-instructions, share of stall samples, active threads), stall attribution\n")
        f.write(txt); f.write("\n# ---- stall samples by reason, top instructions\n"); f.write(st)
    print("wrote", f"profiles/{rnd}_{tag}_{k}.txt")
