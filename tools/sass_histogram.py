#!/usr/bin/env python
"""SASS opcode histogram of the in-tree kernel library, per kernel family -> profiles/sass_<tag>.md

    python tools/sass_histogram.py r02

Evidence for the claims DESIGN.md makes about the instruction mix (wgmma = HGMMA, TMA engine = UBLKCP / UTMALDG / UTMASTG, cp.async = LDGSTS, mbarrier = SYNCS, packed fp32 =
FFMA2 / FADD2 / FMUL2, special function unit = MUFU.EX2, warp reductions = REDUX).  Runs on CPU
(cuobjdump -sass of pvn3d_b200/_build/*.o); the objects are the ones linked into libpvn3d_b200.so.
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "pvn3d_b200", "_build")
WATCH = ["HGMMA", "UTCHMMA", "UTCQMMA", "UTCBAR", "UTCATOMSWS", "LDTM", "STTM", "UTMALDG", "UTMASTG", "UBLKCP", "UTMAPF", "LDGSTS",
         "SYNCS", "HMMA", "MUFU.EX2", "MUFU.RSQ", "MUFU.RCP", "FFMA2", "FADD2", "FMUL2", "REDUX", "SHFL", "ATOMS", "ATOMG",
         "RED", "BAR.SYNC", "MEMBAR", "LDG", "STG", "LDS", "STS", "FFMA", "IMAD"]


def kernels(obj):
    out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
    name, hist = None, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                yield name, hist
            name, hist = m.group(1), collections.Counter()
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if m and hist is not None:
            hist[m.group(1)] += 1
    if name:
        yield name, hist


def demangle(n):
    try:
        return subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip()
    except Exception:
        return n


def main():
    tag = sys.argv[1] if len(sys.argv) > 1 else "r02"
    rows = []
    for f in sorted(os.listdir(OBJ)):
        if not f.endswith(".o"):
            continue
        for name, hist in kernels(os.path.join(OBJ, f)):
            d = demangle(name)
            d = re.sub(r"pvn3d::\(anonymous namespace\)::", "", d)
            d = re.sub(r"\(.*\)$", "", d)
            total = sum(hist.values())
            counts = {}
            for w in WATCH:
                c = sum(v for k, v in hist.items() if k == w or k.startswith(w + "."))
                if w in ("LDG", "STG", "LDS", "STS", "FFMA", "RED"):   # exact family, not prefixes of other opcodes
                    c = sum(v for k, v in hist.items() if k.split(".")[0] == w)
                if c:
                    counts[w] = c
            rows.append((f.replace(".o", ".cu"), d, total, counts))
    lines = [f"# SASS opcode histogram, tag {tag}: `cuobjdump -sass pvn3d_b200/_build/*.o` (sm_90a, the objects linked into libpvn3d_b200.so)",
             "", "Static instruction counts per kernel (not execution counts).  wgmma: HGMMA;",
             "TMA engine: UBLKCP (1-D bulk copy), UTMALDG/UTMASTG (tensor-map loads/stores); cp.async: LDGSTS; mbarrier: SYNCS.", "",
             "| source | kernel | SASS instr | watched opcodes |", "|---|---|---:|---|"]
    for src, d, total, counts in rows:
        lines.append(f"| {src} | `{d[:110]}` | {total} | " + ", ".join(f"{k} {v}" for k, v in counts.items()) + " |")
    agg = collections.Counter()
    for _, _, _, counts in rows:
        agg.update(counts)
    lines += ["", "Library totals: " + ", ".join(f"{k} {agg[k]}" for k in WATCH if agg[k])]
    out = os.path.join(ROOT, "profiles", f"sass_{tag}.md")
    open(out, "w").write("\n".join(lines) + "\n")
    print(out)


if __name__ == "__main__":
    main()
