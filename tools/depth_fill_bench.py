"""Time the GPU fill_missing (DepthFiller) and FrameInputBuilder with and without it; print one JSON line.

Frames: 16 YCB-shape 480x640 box scenes with dropout and holes (synth.make_icp_depth_batch, hole_frac 0.05,
four hole boxes), cam_scale 10000.  Device times are medians of CUDA-event-timed calls after warm-up; a
torch.profiler pass splits the fill into its kernels.  The reference's CPU time (cv2 on the host) is not
measured here: make_golden_fill.log records it.

    python tools/depth_fill_bench.py [--reps 20] [--warmup 3]
"""
import argparse
import json
import os
import re
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pvn3d_b200 import synth  # noqa: E402
from pvn3d_b200.depth_fill import DepthFiller  # noqa: E402
from pvn3d_b200.frame_input import FrameInputBuilder  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from frame_input_bench import gpu_info, timed  # noqa: E402

B, N = 16, 12288


def kernel_times(fn, reps):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        m = re.search(r"(fill_\w+kernel(<\w+>)?)", e.key)
        if m:
            name = m.group(1)
            out[name] = round(out.get(name, 0.0) + e.device_time_total / 1000.0 / reps, 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("depth_fill_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    d = synth.make_icp_depth_batch(B, seed=0, hole_frac=0.05, n_hole_boxes=4)
    rgb = np.random.default_rng(0).integers(0, 256, size=(B, 3, synth.H, synth.W), dtype=np.uint8)
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in
         (("depth", d["depth"]), ("K", d["K"]), ("cam_scale", d["cam_scale"]), ("rgb", rgb))}
    filler = DepthFiller(B, synth.H, synth.W, device=dev)
    fill = lambda: filler.fill(t["depth"], t["cam_scale"])
    plain = FrameInputBuilder(B, N, normals="full", device=dev)
    filled = FrameInputBuilder(B, N, normals="full", fill="multiscale", device=dev)
    build_plain = lambda: plain.build(t["depth"], t["K"], t["cam_scale"], t["rgb"], 1)
    build_filled = lambda: filled.build(t["depth"], t["K"], t["cam_scale"], t["rgb"], 1)
    name, watts = gpu_info()
    out = {"gpu": name, "power_limit_w": watts, "frames": B, "height": synth.H, "width": synth.W,
           "valid_in_mean": round(float((t["depth"] > 0).float().sum((1, 2)).mean()), 1)}
    out["ms_fill"] = round(timed(fill, args.reps, args.warmup), 4)
    out["ms_fill_per_frame"] = round(out["ms_fill"] / B, 4)
    out["valid_out_mean"] = round(float((filler.out > 1e-6).float().sum((1, 2)).mean()), 1)
    out["ms_build_full"] = round(timed(build_plain, args.reps, args.warmup), 4)
    out["ms_build_full_fill"] = round(timed(build_filled, args.reps, args.warmup), 4)
    out["ms_fill_kernels"] = kernel_times(fill, args.reps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
