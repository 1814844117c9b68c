"""Time eval_icp's biggest-cluster filter (flat mean shift, bandwidth 0.06) on the GPU and batched ICP with
and without it, and print one JSON line.

Regime: 16 frames x 5 objects, 2000 labelled scene points per object (1800 on the object with 10 %
outliers, plus a 200-point stray blob 0.2 m beyond the box), box models of 3000 points, ICP max_iter 500,
tol 1e-9, inits 5 deg / 1 cm off the ground truth.  Times are medians of CUDA events after warm-up:
the filter alone (one pvn3d_flat_ms_fit_batch launch over the 80 selections), and IcpRefiner.refine()
without and with cluster_bandwidth.  Not part of bench.py's frame metric.

    python tools/icp_cluster_bench.py [--reps 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import flat_meanshift_oracle as fmo  # noqa: E402
from oracle import icp_oracle  # noqa: E402
from pvn3d_b200 import synth  # noqa: E402
from pvn3d_b200.eval_utils import pose_add_adds  # noqa: E402
from pvn3d_b200.icp import IcpRefiner  # noqa: E402
from pvn3d_b200.meanshift import flat_mean_shift_batch  # noqa: E402

BW = 0.06


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
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return {"median": round(float(np.median(ms)), 3), "min": round(float(np.min(ms)), 3),
            "max": round(float(np.max(ms)), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    data = synth.make_icp_batch(16, 5, 1800, seed=200, model_pts=3000, outlier_frac=0.10, n_stray=200,
                                angle_deg=5.0, offset=0.01)
    b, n, _ = data["pcld"].shape
    t = [torch.from_numpy(np.ascontiguousarray(data[k])).to(dev) for k in ("pcld", "mask", "init", "present")]

    # the filter alone, on the same 80 selections the refiner clusters
    clouds = [data["pcld"][f][icp_oracle.select(data["mask"][f], c, 2000)].astype(np.float64)
              for f in range(b) for c in np.nonzero(data["present"][f])[0]]
    off = np.concatenate([[0], np.cumsum([len(x) for x in clouds])]).astype(np.int32)
    X = torch.from_numpy(np.concatenate(clouds)).to(dev)
    out = {}

    def filt():
        out["r"] = flat_mean_shift_batch(X, off, BW, 300)

    t_filter = timed(filt, a.reps, a.warmup)
    n_iter = out["r"][4].cpu().numpy()
    seeds = np.array([len(fmo.bin_seeds(x, BW)) for x in clouds])

    kw = dict(max_pts=2000, min_pts=1500, max_iter=500, tol=1e-9, device=dev)
    plain = IcpRefiner(data["models"], len(data["models"]), b, n, **kw)
    clus = IcpRefiner(data["models"], len(data["models"]), b, n, cluster_bandwidth=BW, **kw)
    t_plain = timed(lambda: plain.refine(*t), a.reps, a.warmup)
    t_clus = timed(lambda: clus.refine(*t), a.reps, a.warmup)
    kept = clus.cluster_pts.cpu().numpy()[data["present"].astype(bool)]

    def mean_add(ref):
        vals = []
        for f in range(b):
            for c in np.nonzero(data["present"][f])[0]:
                mdl = torch.from_numpy(data["models"][c]).to(dev)
                gt = torch.from_numpy(data["gt"][f, c]).to(dev)
                vals.append(float(pose_add_adds(ref.poses[f, c], gt, mdl)[0][0]))
        return round(float(np.mean(vals)) * 1e3, 3)

    res = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "reps": a.reps,
           "batch": 16, "objects": 5, "scene_pts": 2000, "stray_pts": 200, "outlier_frac": 0.1, "bandwidth": BW,
           "init": "5deg/1cm", "icp_max_iter": 500, "icp_tol": 1e-9, "fits": len(clouds),
           "filter_ms": t_filter, "refine_ms_plain": t_plain, "refine_ms_clustered": t_clus,
           "seeds_mean": round(float(seeds.mean()), 1), "seeds_max": int(seeds.max()),
           "filter_iters_mean": round(float(n_iter.mean()), 1), "filter_iters_max": int(n_iter.max()),
           "kept_pts_mean": round(float(kept.mean()), 1), "kept_pts_min": int(kept.min()),
           "add_mm_plain": mean_add(plain), "add_mm_clustered": mean_add(clus)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
