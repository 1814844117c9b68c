"""Time the batched scoring of a test batch against the reference's per-object scoring; prints ONE JSON line.

    python tools/eval_bench.py [--iters 50]

  add_batch        PoseEvaluator.add_batch on a YCB-shape batch (16 frames x 5 ground-truth objects, 21 synthetic
                   meshes of 2000 points): one pvn3d_frame_add_adds call, CUDA events around `iters` calls
  per_object       what eval_metric does for the same batch: Basic_Utils.cal_add_cuda / cal_adds_cuda
                   (oracle/metrics_oracle.py, the same torch ops) on CUDA per object, each followed by its .item()
  large_mesh       add_batch with one 20000-point mesh (16 frames x 1 object)
  eval_pose_parallel (only where the reference Python is staged under oracle/_ref/py) TorchEval.eval_pose_parallel
                   after compat.install(patch_post=True), the reference's thread pool against patch_eval_pose_parallel,
                   on 16 synthetic YCB frames of 12288 points
The GPU's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import metrics_oracle  # noqa: E402
from pvn3d_b200 import compat, synth  # noqa: E402
from pvn3d_b200.eval_utils import PoseEvaluator  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def timed(fn, iters, dev):
    fn()
    torch.cuda.synchronize(dev)
    t0 = torch.cuda.Event(enable_timing=True)
    t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize(dev)
    return t0.elapsed_time(t1) / iters


def ycb_batch(rng, b, objs, n_cls, p, dev):
    meshes = {c: rng.uniform(-0.08, 0.08, (p, 3)).astype(np.float32) for c in range(1, n_cls)}
    gt = np.zeros((b, 22, 3, 4), np.float32)
    ids = np.zeros((b, 22), np.int32)
    poses = np.zeros((b, n_cls, 3, 4), np.float32)
    for f in range(b):
        cls = rng.permutation(np.arange(1, n_cls))[:objs]
        for i, c in enumerate(cls):
            gt[f, i, :, :3] = synth._haar_rotation(rng)
            gt[f, i, :, 3] = rng.uniform([-0.2, -0.2, 0.6], [0.2, 0.2, 1.0])
            ids[f, i] = c
            poses[f, c] = gt[f, i] + rng.normal(0, 0.01, (3, 4))
    present = (np.abs(poses).sum((2, 3)) > 0).astype(np.uint8)
    t = [torch.from_numpy(x).to(dev) for x in (poses, present, gt, ids)]
    return meshes, t


def per_object(meshes_dev, t):
    poses, present, gt, ids = t
    ids_h = ids.cpu().numpy()                      # eval_metric walks the host-side cls_ids
    out = []
    for f in range(ids_h.shape[0]):
        for i in range(ids_h.shape[1]):
            c = int(ids_h[f, i])
            if c == 0:
                break
            pred = poses[f, c] if present[f, c] else torch.zeros(3, 4, device=poses.device)
            out.append(metrics_oracle.cal_add(pred, gt[f, i], meshes_dev[c]).item())
            out.append(metrics_oracle.cal_adds(pred, gt[f, i], meshes_dev[c]).item())
    return out


def dropin(dev, iters):
    from helpers import load_reference_python

    ref = load_reference_python()
    if ref is None:
        return None
    compat.install(patch_post=True)
    ev = ref.eval_utils
    rng = np.random.default_rng(3)
    for c in range(1, 22):
        ev.bs_utils.ycb_cls_ptsxyz_cuda_dict[ev.cls_lst[c - 1]] = torch.from_numpy(
            rng.uniform(-0.06, 0.06, (2000, 3)).astype(np.float32)).to(dev)
    frames = synth.make_batch("ycb", 16, n_points=12288, config_id=5)
    rts = np.zeros((16, 22, 3, 4), np.float32)
    ids = np.zeros((16, 22, 1), np.int64)
    for f, fr in enumerate(frames):
        rts[f, :len(fr.cls_ids)] = fr.RTs
        ids[f, :len(fr.cls_ids), 0] = fr.cls_ids
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
    masks = t(np.stack([f.labels for f in frames])).long()
    args = (t(np.stack([f.pcld for f in frames])), None, masks, t(np.stack([f.ctr_of for f in frames])), None, masks, 0,
            t(ids), t(rts), t(np.stack([f.kp_of for f in frames])))
    cls = ev.TorchEval
    orig = cls.eval_pose_parallel

    def run():
        te = cls()
        te.eval_pose_parallel(*args, min_cnt=1, use_p2d=False, use_ctr_clus_flter=True, use_ctr=True)
        torch.cuda.synchronize(dev)

    res = {}
    for name in ("reference_ms", "patched_ms"):
        if name == "patched_ms":
            compat.patch_eval_pose_parallel(cls)
        run()
        t0 = time.perf_counter()
        for _ in range(max(1, iters // 10)):
            run()
        res[name] = (time.perf_counter() - t0) * 1e3 / max(1, iters // 10)
    cls.eval_pose_parallel = orig
    res["frames"] = 16
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    meshes, t = ycb_batch(rng, 16, 5, 22, 2000, dev)
    ev = PoseEvaluator(meshes, [13, 16, 19, 20, 21], device=dev)
    meshes_dev = {c: torch.from_numpy(m).to(dev) for c, m in meshes.items()}
    out = {"gpu": gpu_info(), "batch": "16 frames x 5 objects, 21 meshes x 2000 points"}
    out["add_batch_ms"] = timed(lambda: ev.add_batch(*t), a.iters, dev)
    ev.reset()
    ref_vals = per_object(meshes_dev, t)
    add, adds = ev.add_batch(*t)
    ours = np.stack([add.cpu().numpy(), adds.cpu().numpy()], -1)[:, :5].reshape(-1)
    out["max_rel_diff_vs_per_object"] = float(np.max(np.abs(ours - np.asarray(ref_vals)) / np.abs(ref_vals)))
    t0 = time.perf_counter()
    for _ in range(max(1, a.iters // 10)):
        per_object(meshes_dev, t)
    torch.cuda.synchronize(dev)
    out["per_object_ms"] = (time.perf_counter() - t0) * 1e3 / max(1, a.iters // 10)
    big, tb = ycb_batch(np.random.default_rng(1), 16, 1, 2, 20000, dev)
    evb = PoseEvaluator(big, device=dev)
    out["large_mesh"] = "16 frames x 1 object, 20000 points"
    out["large_mesh_add_batch_ms"] = timed(lambda: evb.add_batch(*tb), max(5, a.iters // 5), dev)
    out["eval_pose_parallel"] = dropin(dev, a.iters)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
