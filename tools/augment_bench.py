"""Time the GPU training augmentation (FrameAugmenter: draw + apply) on 24 YCB-shape and 32 LineMOD-shape 480x640
frames; print one JSON line.

Frames: random colour, depth with 30 % holes, half the pixels labelled, a random background frame.  Kinds: YCB
syn frames with real ones mixed in 4:1 (real_syn_gen's split); LineMOD 30 % real, 28 % fuse, 42 % render.  Device
times are medians of CUDA-event-timed draw + apply calls after warm-up; a torch.profiler pass splits the apply by
stage (jitter = luma sums and jitter steps; per noise pass hsv, sharpen, motion, gauss; noise = the noise, the
composite and the output store).  Beside it, the same frame's augmentation as the reference runs it on the CPU
(torchvision's ColorJitter on a PIL image, then rgb_add_noise's cv2 / numpy calls and add_real_back's composite,
every branch of a syn frame on), or "unavailable" when cv2 / PIL / torchvision cannot be imported.

    python tools/augment_bench.py [--reps 20] [--warmup 3]
"""
import argparse
import json
import os
import re
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)
from pvn3d_b200.augment import FrameAugmenter  # noqa: E402
from frame_input_bench import gpu_info, timed  # noqa: E402

H, W = 480, 640
SHAPES = {"ycb": 24, "linemod": 32}
STAGES = (("jitter", r"luma_sum_kernel|jitter_step_kernel"), ("hsv", r"hsv_kernel"), ("sharpen", r"sharpen_kernel"),
          ("motion", r"motion_kernel"), ("gauss", r"gauss_kernel"), ("noise_composite", r"noise_kernel"),
          ("draw", r"augment_draw_kernel"))


def frames(b, seed):
    rng = np.random.default_rng(seed)
    rgb = rng.integers(0, 256, (b, H, W, 3), dtype=np.uint8)
    depth = rng.integers(300, 3000, (b, H, W)).astype(np.float32)
    depth[rng.random((b, H, W)) < 0.3] = 0
    labels = (rng.random((b, H, W)) < 0.5).astype(np.uint8)
    back = rng.integers(0, 256, (b, H, W, 3), dtype=np.uint8)
    back_labels = (rng.random((b, H, W)) < 0.3).astype(np.uint8)
    back_depth = rng.integers(300, 3000, (b, H, W)).astype(np.float32)
    return rgb, depth, labels, back, back_labels, back_depth


def kinds(dataset, b, seed):
    rng = np.random.default_rng(seed)
    if dataset == "ycb":
        return (rng.random(b) <= 0.8).astype(np.int32)
    u = rng.random(b)
    return np.where(u < 0.3, 0, np.where(rng.random(b) < 0.4, 2, 1)).astype(np.int32)


def stage_times(fn, reps):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {k: 0.0 for k, _ in STAGES}
    for e in prof.key_averages():
        for k, pat in STAGES:
            if re.search(pat, e.key):
                out[k] += e.device_time_total / 1000.0 / reps
    return {k: round(v, 4) for k, v in out.items()}


def cpu_frame_ms(reps=5):
    """the reference's augmentation of one YCB syn frame on the CPU, as its calls run it, every branch on"""
    try:
        import cv2
        import torchvision.transforms as transforms
        from PIL import Image
    except ImportError:
        return "unavailable", None
    rgb, depth, labels, back, back_labels, back_depth = (x[0] for x in frames(1, 5))
    rng = np.random.default_rng(6)
    jitter = transforms.ColorJitter(0.2, 0.2, 0.2, 0.05)

    def one():
        img = np.array(jitter(Image.fromarray(rgb)))[:, :, :3]
        for _ in range(2):          # the noise pass, then the composite and the second pass
            hsv = cv2.cvtColor(img, cv2.COLOR_BGR2HSV).astype(np.uint16)
            hsv[:, :, 1] = np.clip(hsv[:, :, 1] * 1.3, 0, 255)
            hsv[:, :, 2] = np.clip(hsv[:, :, 2] * 1.2, 0, 255)
            img = cv2.cvtColor(hsv.astype(np.uint8), cv2.COLOR_HSV2BGR)
            k = -np.ones((3, 3))
            k[1, 1] = 10.5
            img = cv2.filter2D(img, -1, k / k.sum())
            mk = np.zeros((14, 14))
            cv2.line(mk, (7, 7), (13, 10), 1.0)
            img = cv2.filter2D(img, -1, mk / mk.sum())
            img = cv2.GaussianBlur(img, (5, 5), 0.6)
            img = np.clip(img + rng.standard_normal(img.shape) * 12, 0, 255).astype(np.uint8)
            img = np.clip(img + rng.normal(0.0, 7.0, img.shape), 0, 255).astype(np.uint8)
            if _ == 0:
                bk = (back_labels <= 0).astype(np.uint8)
                msk = np.repeat((labels <= 0).astype(np.uint8)[:, :, None], 3, 2)
                img = img * (msk == 0) + back * bk[:, :, None] * msk
                depth_out = np.where(depth > 1e-6, depth, back_depth * bk)
        return img, depth_out

    one()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        one()
        ts.append((time.perf_counter() - t0) * 1e3)
    return round(float(np.median(ts)), 2), f"cv2 {cv2.__version__} ({cv2.getNumThreads()} threads), {os.cpu_count()} cpus"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("augment_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    name, watts = gpu_info()
    res = {"gpu": name, "power_limit_w": watts, "height": H, "width": W}
    for ds, b in SHAPES.items():
        t = [torch.from_numpy(x).to(dev) for x in frames(b, 1)]
        k = torch.from_numpy(kinds(ds, b, 2)).to(dev)
        aug = FrameAugmenter(b, ds, H, W, device=dev)
        seed = [0]

        def step():
            seed[0] += 1
            return aug.apply(*t, aug.draw(seed[0], k))

        ms = timed(step, args.reps, args.warmup)
        res[ds] = {"batch": b, "device_ms_per_batch": round(ms, 4), "device_us_per_frame": round(ms * 1e3 / b, 2),
                   "stages_ms": stage_times(step, 5)}
    cpu_ms, cpu_what = cpu_frame_ms()
    res["reference_cpu_ms_per_ycb_syn_frame"] = cpu_ms
    if cpu_what:
        res["reference_cpu"] = cpu_what
    print(json.dumps(res))


if __name__ == "__main__":
    main()
