"""Summarise ncu artefacts from gpurun_out/ into profiles/ (tracked).

    python tools/summarise_ncu.py r01
writes profiles/launches_<tag>.md (per-kernel share of one bench run, from the
`--metrics gpu__time_duration.sum` launch list) and profiles/<kernel>_<tag>.md (key counters of the
`--set full` captures: duration, DRAM bytes, DRAM %, issue %, pipe %, registers, occupancy).
"""
import collections
import csv
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "profiles")
KEYS = ["launch__grid_size", "launch__block_size", "launch__registers_per_thread", "launch__occupancy_limit_shared_mem",
        "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__inst_executed.sum", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "lts__t_bytes.sum",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_tensor.avg.pct_of_peak_sustained_active",
        "sm__pipe_tensor_subpipe_tmem_cycles_active.avg.pct_of_peak_sustained_active",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum"]


def launches(tag):
    path = os.path.join(ROOT, "gpurun_out", f"launches_{tag}.csv")
    if not os.path.exists(path):
        return
    lines = [l for l in open(path) if not l.startswith("==")]
    agg = collections.defaultdict(lambda: [0, 0.0])
    for r in csv.DictReader(lines):
        if r.get("Metric Name") != "gpu__time_duration.sum":
            continue
        v = float(r["Metric Value"].replace(",", ""))
        u = r["Metric Unit"]
        v = v / 1e3 if u in ("nsecond", "ns") else v * 1e3 if u in ("msecond", "ms") else v * 1e6 if u in ("second", "s") else v
        k = re.sub(r"\(.*", "", r["Kernel Name"])
        k = re.sub(r"<unnamed>::", "", k)[:90]
        agg[k][0] += 1
        agg[k][1] += v
    tot = sum(v for _, v in agg.values())
    with open(os.path.join(OUT, f"launches_{tag}.md"), "w") as f:
        f.write(f"# ncu launch list, tag {tag}: `ncu --metrics gpu__time_duration.sum --clock-control none` over "
                f"`python bench.py --steps 1 --warmup 3 --quick --no-overlap`\n\n"
                f"Per-launch times are cold-cache and serialised: read the SHARES.  {sum(n for n, _ in agg.values())} launches, "
                f"{tot / 1e3:.1f} ms total.\n\n| kernel | launches | total ms | share |\n|---|---:|---:|---:|\n")
        for k, (n, v) in sorted(agg.items(), key=lambda x: -x[1][1])[:30]:
            f.write(f"| `{k}` | {n} | {v / 1e3:.2f} | {100 * v / tot:.1f}% |\n")


def full(tag, name):
    rep = os.path.join(ROOT, "gpurun_out", f"prof_{name}_{tag}.ncu-rep")
    if not os.path.exists(rep):
        return
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rd = list(csv.reader(out.splitlines()))
    hdr, units, rows = rd[0], rd[1], rd[2:]
    with open(os.path.join(OUT, f"ncu_{name}_{tag}.md"), "w") as f:
        kn = hdr.index("Kernel Name") if "Kernel Name" in hdr else None
        f.write(f"# ncu --set full, tag {tag}, kernels matching `{name}` ({len(rows)} launches captured)\n\n")
        if kn is not None:
            f.write("Launches: " + "; ".join(f"{i}: `{re.sub(r'[(].*', '', r[kn])[-60:]}`" for i, r in enumerate(rows)) + "\n\n")
        f.write("| metric | unit | " + " | ".join(f"launch {i}" for i in range(len(rows))) + " |\n")
        f.write("|---|---|" + "---:|" * len(rows) + "\n")
        for k in KEYS:
            if k in hdr:
                i = hdr.index(k)
                f.write(f"| {k} | {units[i]} | " + " | ".join(r[i] for r in rows) + " |\n")


if __name__ == "__main__":
    tag = sys.argv[1] if len(sys.argv) > 1 else "r01"
    os.makedirs(OUT, exist_ok=True)
    launches(tag)
    for name in ("qg", "ms", "mlp", "msdens", "mswit", "fps", "nn", "ball", "glue"):
        gz = os.path.join(ROOT, "gpurun_out", f"prof_{name}_{tag}.ncu-rep.gz")
        if os.path.exists(gz) and not os.path.exists(gz[:-3]):
            subprocess.run(["gunzip", "-kf", gz])
        full(tag, name)
    print(sorted(os.listdir(OUT)))
