"""time of FusedPointnet2MSG.queries() (ball queries of SA1-SA4, 3-NN + weights of FP1-FP4) on a fixed sampling plan, at
the three shapes bench.py runs: ms per call (CUDA events, profiler off), per-launch durations (CUPTI through
torch.profiler, a run of its own), and a checksum of the tables -- run it on two trees to compare them.

    python tools/geo_bench.py [linemod ycb stress]
"""
import collections, hashlib, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import profile, ProfilerActivity
import bench
from pvn3d_b200 import synth, testing
from pvn3d_b200.mlp import FusedPointnet2MSG

dev = torch.device("cuda:0")
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
print("gpu:", torch.cuda.get_device_name(dev), "|", smi.stdout.strip().splitlines()[0] if smi.stdout else "power limit unknown")
eng = FusedPointnet2MSG(testing.seeded_pointnet2msg(0, 1), dev)


def dur(e):
    return e.device_time if hasattr(e, "device_time") else e.cuda_time


def kname(e):
    return e.name.replace("(anonymous namespace)::", "").replace("void ", "").split("(")[0].split("<")[0][-32:]


for name in sys.argv[1:] or list(bench.CONFIGS):
    cfg = bench.CONFIGS[name]
    kw = dict(lm_obj_id=1) if cfg["shape"] == "linemod" else {}
    if cfg.get("n_inst"):
        kw["n_instances"] = cfg["n_inst"]
    frames = synth.make_batch(cfg["shape"], cfg["batch"], n_points=cfg["n_points"], config_id=cfg["config_id"],
                              first_frame=0, **kw)
    cloud = torch.from_numpy(synth.stack(frames)["cld_rgb_nrm"]).to(dev)
    base = eng.sampling(cloud)

    def run():
        base.ball, base.nn = [], {}   # the same sampled levels every call
        return eng.queries(base)

    for _ in range(5):
        run()
    torch.cuda.synchronize()
    n = 50
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        plan = run()
    e1.record()
    torch.cuda.synchronize()
    h = hashlib.sha1()
    for a, b in plan.ball:
        h.update(a.cpu().numpy().tobytes()); h.update(b.cpu().numpy().tobytes())
    for i in range(4):
        h.update(plan.nn[i][0].cpu().numpy().tobytes()); h.update(plan.nn[i][1].cpu().numpy().tobytes())
    print(f"{name} {cfg['batch']}x{cfg['n_points']}: queries() {e0.elapsed_time(e1) / n:.3f} ms/call  "
          f"sha {h.hexdigest()[:12]}")
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            run()
        torch.cuda.synchronize()
    ks = sorted((e for e in prof.events() if e.device_type is not None and "cuda" in str(e.device_type).lower()
                 and e.time_range is not None), key=lambda e: e.time_range.start)
    per = len(ks) // 3
    last = ks[-per:]
    tot = collections.Counter()
    for e in ks:
        tot[kname(e)] += dur(e) / 3
    print(f"  {per} device activities per call, busy {sum(tot.values()):.1f} us, span "
          f"{(last[-1].time_range.start + dur(last[-1]) - last[0].time_range.start):.1f} us")
    for k, v in tot.most_common():
        print(f"    {k:34s} {v:8.1f} us/call")
    print("  launch order (us):", [(kname(e), round(dur(e), 1)) for e in last])
