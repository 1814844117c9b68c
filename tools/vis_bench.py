"""Time demo.py's pose overlay and print ONE JSON line (with the GPU's name and power limit, read in the same run):

  cv2_loop_ms        the reference's way (Basic_Utils.draw_p2ds, basic_utils.py:315-323): one cv2.circle per point of
                     one 2,620-point object on a 480x640 frame, in a Python loop on this host's CPU ("not measured"
                     when cv2 is not installed)
  dropin_ms          vis_utils.draw_p2ds on the same object, host to host: the image and points go to the GPU, are drawn
                     and come back into the caller's arrays
  overlay_us         PoseOverlay.draw on 16 YCB-shape frames (480x640) x 5 objects of 2,620 points, timed with CUDA
                     events; overlay_kernel_us is the device time of its memset and two kernels (torch.profiler)

Host times are medians over --reps calls after --warmup calls (time.perf_counter); device times are medians of
CUDA-event-timed calls.

    python tools/vis_bench.py [--reps 50] [--warmup 5]
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
from pvn3d_b200 import synth, vis_utils  # noqa: E402
from pvn3d_b200.vis_utils import PoseOverlay  # noqa: E402

H, W, N_PTS, B, OBJS, N_CLS = 480, 640, 2620, 16, 5, 22
K_YCB = np.array([[1066.778, 0.0, 312.9869], [0.0, 1067.487, 241.3109], [0.0, 0.0, 1.0]], np.float32).astype(np.float64)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, watts = (s.strip() for s in out.splitlines()[0].split(","))
        return name, float(watts)
    except Exception:  # noqa: BLE001 -- reported as unknown
        return torch.cuda.get_device_name(0), None


def host_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return round(float(np.median(ts)), 3)


def device_us(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return round(float(np.median(ts)), 1)


def kernel_us(fn, names):
    """device time (us) of the work whose name contains one of `names` in one call of fn (torch.profiler)"""
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = 0.0
    for e in prof.key_averages():
        if any(n in e.key for n in names):
            tot += getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0.0)
    return round(tot, 1)


def mesh(rng, n=N_PTS):
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return (d * rng.uniform(0.03, 0.07, 3)).astype(np.float32)


def project(pts, pose):
    """demo.py's transform and project_p3d (float64), as int32 pixel coordinates"""
    p = np.dot(pts, pose[:, :3].T) + pose[:, 3]
    q = np.dot(p, K_YCB.T)
    q[q[:, 2] < 1e-8, 2] = 1.0
    return np.around(q[:, :2] / q[:, 2:]).astype(np.int32)


def cv2_loop(img, p2ds, r, color):
    """the reference's per-point loop (basic_utils.py:315-323), restated"""
    import cv2

    h, w = img.shape[:2]
    for pt in p2ds:
        pt[0] = np.clip(pt[0], 0, w)
        pt[1] = np.clip(pt[1], 0, h)
        img = cv2.circle(img, (int(pt[0]), int(pt[1])), r, color, -1)
    return img


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vis_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    name, watts = gpu_info()
    rng = np.random.default_rng(7)
    pose = np.concatenate([synth._haar_rotation(rng), np.array([[0.0], [0.0], [0.8]])], 1)
    obj = mesh(rng)
    p2ds = project(obj, pose)
    bg = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    color = (0, 115, 87)
    res = {"gpu": name, "power_limit_w": watts, "frame": [H, W], "points_per_object": N_PTS}
    try:
        import cv2  # noqa: F401

        res["cv2_loop_ms"] = host_ms(lambda: cv2_loop(bg.copy(), p2ds.copy(), 1, color), max(5, args.reps // 5), 2)
        a = cv2_loop(bg.copy(), p2ds.copy(), 1, color)
        b = vis_utils.draw_p2ds(bg.copy(), p2ds.copy(), 1, color)
        res["dropin_equals_cv2_loop"] = bool(np.array_equal(a, b))
    except ImportError:
        res["cv2_loop_ms"] = "not measured"
    res["dropin_ms"] = host_ms(lambda: vis_utils.draw_p2ds(bg.copy(), p2ds.copy(), 1, color), args.reps, args.warmup)
    # the batched overlay: 16 frames x 5 of 21 classes
    meshes = {c: mesh(rng) for c in range(1, N_CLS)}
    ov = PoseOverlay(meshes, dev)
    poses = np.zeros((B, N_CLS, 3, 4))
    present = np.zeros((B, N_CLS), np.uint8)
    order = np.zeros((B, N_CLS), np.int32)
    for f in range(B):
        ids = rng.choice(np.arange(1, N_CLS), OBJS, replace=False)
        order[f, :OBJS] = ids
        for j, c in enumerate(ids):
            poses[f, c] = np.concatenate([synth._haar_rotation(rng),
                                          np.array([[-0.12 + 0.06 * j], [rng.uniform(-0.05, 0.05)], [0.8]])], 1)
            present[f, c] = 1
    imgs = torch.from_numpy(rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)).to(dev)
    t = [torch.from_numpy(x).to(dev) for x in (poses, present, order, K_YCB)]
    colors = torch.from_numpy(vis_utils.label_colors(N_CLS)).to(dev)
    work = imgs.clone()
    fn = lambda: ov.draw(work, t[0], t[1], t[2], t[3], colors)   # noqa: E731
    res["overlay_frames"], res["overlay_objects_per_frame"] = B, OBJS
    res["overlay_us"] = device_us(fn, args.reps, args.warmup)
    res["overlay_kernel_us"] = kernel_us(fn, ["vis_mark", "vis_paint", "Memset"])
    res["overlay_us_per_frame"] = round(res["overlay_us"] / B, 2)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
