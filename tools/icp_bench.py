"""Time batched ICP refinement (IcpRefiner) in pvn3d/eval_icp.py's regime and print one JSON line.

16 frames x 5 objects, 2000 scene points per object, box models of 3000 points, max_iter 500,
tol 1e-9, inits 5 deg / 1 cm and 15 deg / 2 cm off the ground truth.  Times come from CUDA events
around refine() after warm-up; not part of bench.py's frame metric.

    python tools/icp_bench.py [--reps 30] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pvn3d_b200 import synth  # noqa: E402
from pvn3d_b200.icp import IcpRefiner  # noqa: E402


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:  # noqa: BLE001 -- reported as unknown
        return None


def run(angle, offset, reps, warmup, dev):
    data = synth.make_icp_batch(16, 5, 2000, seed=100 + int(angle), model_pts=3000, angle_deg=angle, offset=offset)
    b, n, _ = data["pcld"].shape
    ref = IcpRefiner(data["models"], len(data["models"]), b, n, max_pts=2000, min_pts=1500, max_iter=500, tol=1e-9,
                     device=dev)
    t = {k: torch.from_numpy(np.ascontiguousarray(data[k])).to(dev) for k in ("pcld", "mask", "init", "present")}
    for _ in range(warmup):
        ref.refine(t["pcld"], t["mask"], t["init"], t["present"])
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _, iters, _, refined = ref.refine(t["pcld"], t["mask"], t["init"], t["present"])
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    it = iters.cpu().numpy()[refined.cpu().numpy().astype(bool)]
    queries = int(((it + 1) * 2000).sum())          # every fit holds exactly 2000 scene points
    tests = ref.pair_tests()
    med = float(np.median(ms))
    return {"init": f"{angle:g}deg/{offset * 100:g}cm", "fits": int(len(it)), "refine_ms_median": round(med, 3),
            "refine_ms_min": round(float(np.min(ms)), 3), "refine_ms_max": round(float(np.max(ms)), 3),
            "iters_mean": round(float(it.mean()), 2), "iters_max": int(it.max()),
            "nn_queries_per_s": float(f"{queries / (med * 1e-3):.4g}"),
            "pair_tests_per_s": float(f"{tests / (med * 1e-3):.4g}"), "pair_tests_per_query": round(tests / queries, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    res = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "reps": a.reps,
           "batch": 16, "objects": 5, "scene_pts": 2000, "model_pts": 3000, "max_iter": 500, "tol": 1e-9,
           "runs": [run(5.0, 0.01, a.reps, a.warmup, dev), run(15.0, 0.02, a.reps, a.warmup, dev)]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
