"""Time eval_icp's full-resolution refinement (DepthIcpRefiner) stage by stage and print one JSON line.

Regime: 16 frames x 5 objects, 480x640 depth with holes (synth.make_icp_depth_batch), 12288 sampled
points with border-flipped labels, eval_icp's settings (max_pts 2000, min_pts 1500, MeanShift
bandwidth 0.06, max_iter 500, tol 1e-9), inits 5 deg / 1 cm off the ground truth.  Times are medians of
CUDA events after warm-up: back-projection, label fill (the per-frame grid build + the search), the
clustered refine, and the whole refine() call; torch.profiler splits the fill's device time into the
grid build and the search.  Mean ADD over the fitted objects before and after.  Not part of bench.py.

    python tools/icp_depth_bench.py [--reps 10] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pvn3d_b200 import fixtures, synth  # noqa: E402
from pvn3d_b200.eval_utils import pose_add_adds  # noqa: E402
from pvn3d_b200.icp import DepthIcpRefiner, depth_to_cloud, fill_label  # noqa: E402


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:  # noqa: BLE001 -- reported as unknown
        return None


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    n_cls, batch = fixtures.YCB_N_CLASSES, 16
    d = synth.make_icp_depth_batch(batch, seed=2026)
    t = {k: torch.from_numpy(np.ascontiguousarray(d[k])).to(dev)
         for k in ("depth", "K", "cam_scale", "init", "present", "pcld", "labels")}
    ref = DepthIcpRefiner(d["models"], n_cls, batch, device=dev)
    cloud, valid = ref.cloud, ref.valid
    run_all = lambda: ref.refine(t["depth"], t["K"], t["cam_scale"], t["init"], t["present"], pcld=t["pcld"],
                                 point_labels=t["labels"])
    run_all()
    torch.cuda.synchronize()
    ms_depth = timed(lambda: depth_to_cloud(t["depth"], t["K"], t["cam_scale"], out=(cloud, valid)), args.reps,
                     args.warmup)
    ms_fill = timed(lambda: fill_label(cloud, valid, t["pcld"], t["labels"], out=ref.labels), args.reps, args.warmup)
    ms_refine = timed(lambda: ref.icp.refine(cloud, ref.labels, t["init"], t["present"]), args.reps, args.warmup)
    ms_total = timed(run_all, args.reps, args.warmup)

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            fill_label(cloud, valid, t["pcld"], t["labels"], out=ref.labels)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        for key in ("icp_build_kernel", "label_fill_kernel", "label_fill_setup_kernel"):
            if key in e.key:
                kern[key] = kern.get(key, 0.0) + e.device_time_total / 1000.0 / args.reps

    poses, iters, err, refined = (x.cpu() for x in run_all())
    before, after, n_fit = [], [], 0
    for b in range(batch):
        for c in np.nonzero(d["present"][b])[0]:
            if not int(refined[b, c]):
                continue
            mdl = torch.from_numpy(d["models"][c]).to(dev)
            gt = torch.from_numpy(d["gt"][b, c]).to(dev)
            before.append(float(pose_add_adds(torch.from_numpy(d["init"][b, c]).to(dev), gt, mdl)[0][0]))
            after.append(float(pose_add_adds(poses[b, c].to(dev), gt, mdl)[0][0]))
            n_fit += 1
    print(json.dumps({
        "gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(),
        "frames": batch, "objects": int(d["present"].sum()), "fits": n_fit, "pixels": 480 * 640,
        "valid_pixels_mean": float(valid.float().sum(1).mean()), "samples": int(d["pcld"].shape[1]),
        "ms_depth_to_cloud": round(ms_depth, 4), "ms_fill_label": round(ms_fill, 4),
        "ms_fill_grid_build": round(kern.get("icp_build_kernel", float("nan")), 4),
        "ms_fill_search": round(kern.get("label_fill_kernel", float("nan")), 4),
        "ms_refine_clustered": round(ms_refine, 4), "ms_total": round(ms_total, 4),
        "iters_mean": float(iters[refined.bool()].float().mean()), "cluster_pts_mean":
            float(ref.cluster_pts.cpu()[refined.bool()].float().mean()),
        "add_mean_before_m": float(np.mean(before)), "add_mean_after_m": float(np.mean(after)),
    }))


if __name__ == "__main__":
    main()
