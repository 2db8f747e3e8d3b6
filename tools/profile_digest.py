#!/usr/bin/env python3
"""Turn gpurun_out/launches_<tag>.csv (ncu --metrics gpu__time_duration.sum launch list of
tools/profile.sh) and gpurun_out/prof_<tag>_<kernel>.ncu-rep (ncu --set full captures) into the
tracked summaries under profiles/.   usage: profile_digest.py <tag> [round]"""
import csv, json, os, re, subprocess, sys, io
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
tag = sys.argv[1]; rnd = sys.argv[2] if len(sys.argv) > 2 else "r01"
src = os.path.join(ROOT, "gpurun_out", f"launches_{tag}.csv")
rows = [r for r in csv.reader(open(src)) if r and r[0].isdigit()]
per = {}; order = []
for r in rows:
    name = re.sub(r"\(.*", "", r[4]).replace("void ", "").replace("b200::", "")
    ns = float(r[14])
    if name not in per: per[name] = [0, 0.0, r[8], r[7]]; order.append(name)
    per[name][0] += 1; per[name][1] += ns
tot = sum(v[1] for v in per.values())
os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)      # git-ignored output directory
out = os.path.join(ROOT, "profiles", f"{rnd}_launches_{tag}.md")
with open(out, "w") as f:
    f.write(f"# ncu launch list `{tag}` (`tools/profile.sh {tag}`: bench.py --batch 16 --steps 1 --warmup 1, every launch, "
            "`--metrics gpu__time_duration.sum --clock-control none`)\n\n")
    f.write("Per-launch times under ncu are cold-cache and serialised: compare SHARES, not absolutes.\n\n")
    f.write("| kernel | launches | total us | share | grid (last) | block |\n|---|---|---|---|---|---|\n")
    for name in sorted(per, key=lambda k: -per[k][1]):
        n, ns, grid, blk = per[name]
        f.write(f"| `{name}` | {n} | {ns / 1e3:.1f} | {ns / tot * 100:.1f} % | {grid} | {blk} |\n")
    f.write(f"\nTotal device time in kernels: {tot / 1e6:.3f} ms over {len(rows)} launches.\n")
print(open(out).read())
import shutil
shutil.copy(src, os.path.join(ROOT, "profiles", f"{rnd}_launches_{tag}.csv"))
# full-set captures
for fn in sorted(os.listdir(os.path.join(ROOT, "gpurun_out"))):
    m = re.match(rf"prof_{tag}_(.+)\.ncu-rep$", fn)
    if not m: continue
    k = m.group(1)
    txt = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ncu_summary.py"), os.path.join(ROOT, "gpurun_out", fn)], capture_output=True, text=True).stdout
    with open(os.path.join(ROOT, "profiles", f"{rnd}_{tag}_{k}.txt"), "w") as f:
        f.write(f"# ncu --set full --clock-control none --import-source on, kernel {k}, capture {tag} (batch 16 of 3840x2160, one launch)\n"
                "# headline metrics, then hot SASS regions (instruction index range, #instr, executions per instr, share of warp-instructions, share of stall samples, active threads)\n")
        f.write(txt)
    print("wrote", f"profiles/{rnd}_{tag}_{k}.txt")
