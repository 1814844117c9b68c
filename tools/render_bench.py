"""Time MeshRenderer.render (csrc/render.cu) on LineMOD-shape batches and print ONE JSON line.

    python tools/render_bench.py [--batch 32] [--iters 20] [--warmup 3]

32 frames of 480x640 with LineMOD's K.  Procedural meshes of about 10 k and 100 k faces (jittered boxes, 12 n^2
faces), objects 0.12 m across at 0.5-1.0 m: `render` puts one object in each frame, `fuse` four objects of different
classes.  Device time per batch from CUDA events (median of --iters calls after --warmup), per frame = per batch /
batch.  For context, the numpy restatement of the same contract (tests/render_ref.py) on one frame, on the host CPU.
The GPU name and power limit are recorded beside the numbers.
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

import render_ref as R  # noqa: E402
from pvn3d_b200.render import MeshRenderer, pack_meshes  # noqa: E402

H, W = 480, 640


def _gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        power = r.stdout.strip().splitlines()[0] if r.returncode == 0 else None
    except (OSError, subprocess.SubprocessError):
        power = None
    return name, power


def _meshes(n, rng, n_cls=5):
    out = {}
    for c in range(1, n_cls):
        v, f, col = R.box(np.array([0.06, 0.05, 0.04]), n, rng)
        v = v + rng.normal(0, 5e-4, v.shape).astype(np.float32)
        out[c] = (v, f, col)
    return out


def _poses(batch, n_cls, per_frame, rng):
    poses = np.zeros((batch, n_cls, 3, 4))
    present = np.zeros((batch, n_cls), np.uint8)
    for f in range(batch):
        classes = rng.choice(np.arange(1, n_cls), per_frame, replace=False)
        for i, c in enumerate(classes):
            off = np.array([[-0.08, -0.06], [0.08, -0.06], [-0.08, 0.06], [0.08, 0.06]])[i] if per_frame > 1 else 0
            t = (*(rng.uniform(-0.03, 0.03, 2) + off), rng.uniform(0.5, 1.0))
            poses[f, c] = R.pose(*rng.uniform(-np.pi, np.pi, 3), t)
            present[f, c] = 1
    return poses, present


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("render_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    name, power = _gpu_info()
    rng = np.random.default_rng(0)
    K = torch.from_numpy(R.LM_K).to(dev)
    res = {"bench": "render", "gpu": name, "power_limit": power, "batch": a.batch, "height": H, "width": W,
           "iters": a.iters, "cases": []}
    for n in (29, 91):                                                   # 10,092 and 99,372 faces per mesh
        meshes = _meshes(n, rng)
        rr = MeshRenderer(meshes, a.batch, H, W, device=dev)
        faces = int(meshes[1][1].shape[0])
        for kind, per in (("render", 1), ("fuse", 4)):
            poses, present = _poses(a.batch, rr.n_cls, per, rng)
            ps, pr = torch.from_numpy(poses).to(dev), torch.from_numpy(present).to(dev)
            for _ in range(a.warmup):
                out = rr.render(ps, pr, K)
            times = []
            for _ in range(a.iters):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = rr.render(ps, pr, K)
                e1.record()
                e1.synchronize()
                times.append(e0.elapsed_time(e1))
            ms = float(np.median(times))
            covered = float((out[2] > 0).float().mean())
            t0 = time.perf_counter()
            R.raster(*pack_meshes(meshes), poses[:1], present[:1], R.LM_K, H, W)
            host = (time.perf_counter() - t0) * 1e3
            res["cases"].append({"kind": kind, "faces_per_mesh": faces, "objects_per_frame": per,
                                 "ms_per_batch": round(ms, 4), "ms_per_frame": round(ms / a.batch, 5),
                                 "ms_min": round(float(np.min(times)), 4), "covered_share": round(covered, 4),
                                 "numpy_ms_per_frame": round(host, 1)})
        del rr
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
