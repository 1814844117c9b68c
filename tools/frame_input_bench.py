"""Time FrameInputBuilder.build() stage by stage and print one JSON line.

Regimes:
  linemod  32 frames, 480x640, two spheres over a plane (synth._render, depth in mm, cam_scale 1000, every pixel
           valid), 12288 points, normals="sampled" (linemod_dataset.py estimates normals on the sampled cloud);
  ycb      16 box scenes with holes (synth.make_icp_depth_batch, ~300 k valid pixels per frame), 12288 points,
           normals="full" (ycb_dataset.py estimates normals on the whole cloud).
Device times are medians of CUDA-event-timed build() calls after warm-up; torch.profiler splits the device
time into back-projection, sampling (select + compact), assembly, grid build (memset + five grid kernels) and
kNN + normals.  The CPU stand-in is the float64 numpy/scipy reference of tests/normals_ref.py (cKDTree
candidates, re-ranked) for one frame on the host cores: PCL itself is not available to time.

    python tools/frame_input_bench.py [--reps 10] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from pvn3d_b200 import synth  # noqa: E402
from pvn3d_b200.frame_input import FrameInputBuilder  # noqa: E402

N = 12288
STAGES = {"depth_to_cloud": ("depth_to_cloud_kernel",), "sampling": ("sample_select_kernel", "sample_compact_kernel"),
          "assembly": ("assemble_kernel",), "grid_build": ("grid_", "Memset"), "knn_normals": ("knn_normals_kernel",)}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, watts = (s.strip() for s in out.splitlines()[0].split(","))
        return name, float(watts)
    except Exception:  # noqa: BLE001 -- reported as unknown
        return torch.cuda.get_device_name(0), None


def linemod_frames(batch, seed=0):
    rng = np.random.default_rng(seed)
    K = synth.K_LINEMOD
    depth = np.zeros((batch, synth.H, synth.W), np.float32)
    for b in range(batch):
        centres = [np.array([rng.uniform(-0.1, 0.1), rng.uniform(-0.05, 0.05), rng.uniform(0.6, 0.9)]) for _ in range(2)]
        d, _ = synth._render(K, centres, [0.05, 0.08], rng)
        depth[b] = np.round(d * 1000.0)
    return dict(depth=depth, K=np.repeat(K.astype(np.float32)[None], batch, 0),
                cam_scale=np.full(batch, 1000.0, np.float32),
                rgb=rng.integers(0, 256, size=(batch, 3, synth.H, synth.W), dtype=np.uint8))


def ycb_frames(batch, seed=0):
    d = synth.make_icp_depth_batch(batch, seed=seed)
    d["rgb"] = np.random.default_rng(seed).integers(0, 256, size=(batch, 3, synth.H, synth.W), dtype=np.uint8)
    return d


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


def stage_times(fn, reps):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in STAGES}
    for e in prof.key_averages():
        for stage, keys in STAGES.items():
            if any(k in e.key for k in keys):
                out[stage] += e.device_time_total / 1000.0 / reps
    return {f"ms_{k}": round(v, 4) for k, v in out.items()}


def cpu_standin_s(d, mode):
    """one frame through the float64 host reference: back-projection, sampling, kNN, normals"""
    import normals_ref as nr
    from oracle import depth_icp_oracle as dio

    t0 = time.perf_counter()
    cloud, valid = dio.dpt_2_cld(d["depth"][0], d["cam_scale"][0], d["K"][0])
    choose, _ = nr.sample_frame(valid, N, 1, 0)
    q = cloud[choose]
    idx = nr.knn(cloud, q, valid) if mode == "full" else nr.knn(q, q)
    nr.normals(cloud if mode == "full" else q, idx, q)
    return time.perf_counter() - t0


def regime(name, d, mode, dev, reps, warmup):
    b = len(d["depth"])
    t = {k: torch.from_numpy(np.ascontiguousarray(d[k])).to(dev) for k in ("depth", "K", "cam_scale", "rgb")}
    fib = FrameInputBuilder(b, N, normals=mode, device=dev)
    run = lambda: fib.build(t["depth"], t["K"], t["cam_scale"], t["rgb"], 1)
    ms = timed(run, reps, warmup)
    res = {"frames": b, "points": N, "normals": mode, "valid_pixels_mean": round(float(fib.valid.float().sum(1).mean()), 1),
           "frames_ok": int(fib.ok.sum()), "ms_build": round(ms, 4), "ms_build_per_frame": round(ms / b, 4)}
    res.update(stage_times(run, reps))
    res["cpu_standin_s_per_frame"] = round(cpu_standin_s(d, mode), 3)
    return name, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("frame_input_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    name, watts = gpu_info()
    out = {"gpu": name, "power_limit_w": watts,
           "cpu_standin": "tests/normals_ref.py (numpy/scipy float64, cKDTree) on %d host cores, not PCL" % os.cpu_count()}
    for key, d, mode in (("linemod_b32", linemod_frames(32), "sampled"), ("ycb_b16", ycb_frames(16), "full")):
        k, res = regime(key, d, mode, dev, args.reps, args.warmup)
        out[k] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
