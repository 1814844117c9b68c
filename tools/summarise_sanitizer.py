"""gpurun_out/sanitizer_<tool>_<suite>_<tag>.log -> profiles/sanitizer_<tag>.md"""
import glob
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
tag = sys.argv[1] if len(sys.argv) > 1 else "r02"
rows = []
for f in sorted(glob.glob(os.path.join(ROOT, "gpurun_out", f"sanitizer_*_{tag}.log"))):
    m = re.match(rf"sanitizer_(\w+?)_(\w+)_{tag}\.log", os.path.basename(f))
    txt = open(f).read()
    tests = re.findall(r"(\d+ (?:passed|failed)[^\n]*)", txt)
    summ = re.findall(r"(ERROR SUMMARY: [^\n]*|RACECHECK SUMMARY: [^\n]*)", txt)
    rows.append((m.group(1), m.group(2), tests[-1] if tests else "?", summ[-1] if summ else "?"))
out = [f"# compute-sanitizer, tag {tag} (`tools/sanitizer_r02.sh` on the GPU)", "",
       "Small-shape selections of the GPU parity tests (the tools slow kernels down 10-100x): MLP = per-layer kernel",
       "(dense / SA-gather / FP-interp producers, store and max-pool epilogues, 1 and 2 CTAs per SM, TMA weights);",
       "ms = mean-shift in all four modes (witness + fallback + cooperative sweep), cal_frame_poses_lm,",
       "Kabsch, ADD/ADD-S, seg argmax; pn2 = three_nn, ball_query, FPS, gathers.", "",
       "| tool | suite | pytest | sanitizer summary |", "|---|---|---|---|"]
for r in rows:
    out.append("| " + " | ".join(r) + " |")
note = os.path.join(ROOT, "profiles", f"sanitizer_{tag}_notes.txt")
if os.path.exists(note):
    out += ["", open(note).read().strip()]
open(os.path.join(ROOT, "profiles", f"sanitizer_{tag}.md"), "w").write("\n".join(out) + "\n")
print("\n".join(out))
