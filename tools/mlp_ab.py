"""shared-MLP time of one 32-frame batch (FusedPointnet2MSG.features on a fixed geometry plan): total ms per call,
output checksum, per-launch durations (CUPTI) -- run it on two trees to compare them"""
import os, sys, hashlib
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pvn3d_b200 import synth, testing
from pvn3d_b200.mlp import FusedPointnet2MSG

dev = torch.device("cuda:0")
B = int(os.environ.get("AB_BATCH", 32))
host = synth.stack(synth.make_batch("linemod", B, config_id=2, lm_obj_id=1))
cloud = torch.from_numpy(host["cld_rgb_nrm"]).to(dev)
eng = FusedPointnet2MSG(testing.seeded_pointnet2msg(0, 1), dev)
plan = eng.geometry(cloud)
for _ in range(3):
    out = eng.features(cloud, plan)
torch.cuda.synchronize()
n = 20
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(n):
    out = eng.features(cloud, plan)
e1.record()
torch.cuda.synchronize()
print(f"features: {e0.elapsed_time(e1) / n:.3f} ms  sha {hashlib.sha1(out.cpu().numpy().tobytes()).hexdigest()[:12]}")
if os.environ.get("AB_LAUNCHES", "1") == "1":
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.features(cloud, plan)
        torch.cuda.synchronize()
    ks = [e for e in prof.events() if any(k in e.name for k in ("mlp_layer_kernel", "mlp_sa_fact2_kernel", "mlp_sa_fact2w_kernel", "mlp_fp2_kernel",
                                                                  "mlp_fp_fact2_kernel"))]
    ks.sort(key=lambda e: e.time_range.start)
    print("  launches us:", [round(e.device_time if hasattr(e, "device_time") else e.cuda_time) for e in ks], "sum",
          round(sum((e.device_time if hasattr(e, "device_time") else e.cuda_time) for e in ks)))
