"""What deterministic mode costs: prints ONE JSON line.

  * grads: each PointNet++ grad op's backward at the training shapes (24 frames x 12288 points, device FPS / ball query
    / three_nn plans), today's atomic entry point against the fixed-order one (`_ext` with
    torch.use_deterministic_algorithms off / on);
  * psp: the prior pools (60x80 -> 2, 3, 6 at 512 channels; the 1x1 prior is torch's mean in both modes), the four
    prior upsamplings (-> 60x80) and up_1 / up_2 / up_3 (x2, align_corners) at B = 24 for resnet34 with
    psp_size = 512: torch's atomic backward against the ordered kernels;
  * step: one training step (forward, model_fn's three losses, backward) of the staged reference PVN3D (resnet34,
    pretrained=False) at B = 2, 480 x 640, N = 12288, with deterministic mode off (the reference's own ops) and on
    (compat.install(patch_deterministic=True), CUBLAS_WORKSPACE_CONFIG=:4096:8); "not measured" when the reference
    Python is not staged under oracle/_ref/py.  Each mode also reports its device time per step summed over kernels and
    its eight largest kernels (torch.profiler, two steps after the timed ones).

Times are CUDA-event medians of `--reps` calls after `--warmup`, in milliseconds.

    python tools/determinism_bench.py [--reps 20] [--warmup 3]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from pvn3d_b200 import _ext, deterministic, synth  # noqa: E402

B, N = 24, 12288
SA_LEVELS = [(12288, 2048, (0.0175, 0.025), (16, 32)), (2048, 1024, (0.025, 0.05), (16, 32)),
             (1024, 512, (0.05, 0.1), (16, 32)), (512, 128, (0.1, 0.2), (16, 32))]
SA_C = (6, 96, 256, 512)
FP_C = (256, 512, 512, 1024)


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
    return round(statistics.median(ts), 4)


def both(fn, reps, warmup):
    """(atomic ms, ordered ms) of fn with deterministic mode off / on"""
    off = timed(fn, reps, warmup)
    torch.use_deterministic_algorithms(True)
    try:
        on = timed(fn, reps, warmup)
    finally:
        torch.use_deterministic_algorithms(False)
    return {"atomic_ms": off, "ordered_ms": on, "ratio": round(on / off, 2)}


def grads(dev, reps, warmup):
    frames = synth.make_batch("ycb", B, n_points=N, config_id=31)
    xyz = torch.from_numpy(np.stack([f.pcld for f in frames])).to(dev).contiguous()
    levels, fps = [xyz], []
    for _, m, _, _ in SA_LEVELS:
        fps.append(_ext.furthest_point_sampling(levels[-1], m))
        levels.append(_ext.gather_xyz(levels[-1], fps[-1]))
    gen = torch.Generator(device=dev).manual_seed(0)
    res = {}
    for li, (n, m, radii, nss) in enumerate(SA_LEVELS):
        for r, ns in zip(radii, nss):
            idx = _ext.ball_query(levels[li + 1], levels[li], r, ns)
            g = torch.randn((B, SA_C[li], m, ns), generator=gen, device=dev)
            # bytes the ordered path must move: grad_out and idx read, grad_points written
            res[f"group_SA{li + 1}_ns{ns}"] = {**both(lambda: _ext.group_points_grad(g, idx, n), reps, warmup),
                                               "mb": round((g.numel() * 4 + idx.numel() * 4 + B * SA_C[li] * n * 4)
                                                           / 1e6, 1)}
        g = torch.randn((B, 3, m), generator=gen, device=dev)
        res[f"gather_SA{li + 1}_c3"] = both(lambda: _ext.gather_points_grad(g, fps[li], n), reps, warmup)
    for lu in range(4):
        d2, idx = _ext.three_nn(levels[lu], levels[lu + 1])
        recip = 1.0 / (torch.sqrt(d2) + 1e-8)
        w = (recip / recip.sum(2, keepdim=True)).contiguous()
        n, m = levels[lu].size(1), levels[lu + 1].size(1)
        g = torch.randn((B, FP_C[lu], n), generator=gen, device=dev)
        res[f"interp_FP{lu + 1}"] = {**both(lambda: _ext.three_interpolate_grad(g, idx, w, m), reps, warmup),
                                     "mb": round((g.numel() * 4 + idx.numel() * 8 + B * FP_C[lu] * m * 4) / 1e6, 1)}
    return res


def psp(dev, reps, warmup):
    gen = torch.Generator(device=dev).manual_seed(1)
    res = {}

    def case(name, x_shape, fwd):
        x = torch.randn(x_shape, generator=gen, device=dev).requires_grad_(True)
        y = fwd(x)
        g = torch.randn(y.shape, generator=gen, device=dev)
        res[name] = both(lambda: torch.autograd.grad(y, x, g, retain_graph=True), reps, warmup)

    for s in (2, 3, 6):       # the 1x1 prior runs torch's mean in both modes
        case(f"pool_60x80_to_{s}", (B, 512, 60, 80), lambda x, s=s: deterministic.adaptive_avg_pool2d(x, (s, s)))
    for s in (1, 2, 3, 6):
        case(f"upsample_{s}_to_60x80", (B, 512, s, s),
             lambda x: deterministic.interpolate(x, size=(60, 80), mode="bilinear", align_corners=False))
    for name, c, h, w in (("up_1", 1024, 60, 80), ("up_2", 256, 120, 160), ("up_3", 64, 240, 320)):
        case(f"{name}_{h}x{w}_x2", (B, c, h, w),
             lambda x: deterministic.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True))
    return res


STEP = r"""
import json, statistics, sys
import torch
sys.path.insert(0, sys.argv[2]); sys.path.insert(0, sys.argv[2] + "/tests")
from helpers import load_reference_python
from pvn3d_b200 import compat
det = sys.argv[1] == "on"
assert load_reference_python() is not None
if det:
    compat.install(patch_deterministic=True)
    torch.use_deterministic_algorithms(True)
import lib.pvn3d as P
from lib.loss import FocalLoss, OFLoss
from lib.pspnet import Modified_PSPNet
P.modified_psp_models["resnet34"] = lambda: Modified_PSPNet(sizes=(1, 2, 3, 6), psp_size=512, deep_features_size=256,
                                                            backend="resnet34", pretrained=False)
dev = torch.device("cuda:0")
torch.manual_seed(0)
model = P.PVN3D(num_classes=22, pcld_input_channels=6, pcld_use_xyz=True, num_kps=8, num_points=12288).to(dev).train()
crit, crit_of = FocalLoss(gamma=2), OFLoss()
b, n = 2, 12288
gen = torch.Generator().manual_seed(1)
rgb = torch.rand((b, 3, 480, 640), generator=gen).to(dev)
cld = torch.randn((b, n, 9), generator=gen).to(dev) * 0.1
choose = torch.stack([torch.randperm(480 * 640, generator=gen)[:n] for _ in range(b)])[:, None].to(dev)
labels = torch.randint(0, 22, (b, n), generator=gen).to(dev)
kp = torch.randn((b, n, 8, 3), generator=gen).to(dev) * 0.05
ctr = torch.randn((b, n, 1, 3), generator=gen).to(dev) * 0.05
def step():
    model.zero_grad(set_to_none=True)
    pk, ps, pc = model(cld, rgb, choose)
    loss = crit(ps.view(labels.numel(), -1), labels.view(-1)).sum() * 2.0 + crit_of(pk, kp, labels).sum() \
        + crit_of(pc, ctr, labels).sum()
    loss.backward()
reps, warmup = int(sys.argv[3]), int(sys.argv[4])
for _ in range(warmup):
    step()
ts = []
for _ in range(reps):
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); step(); e.record(); e.synchronize()
    ts.append(a.elapsed_time(e))
# where the step's GPU time goes: device time per kernel name over two profiled steps, per step
from torch.profiler import ProfilerActivity, profile
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(2):
        step()
    torch.cuda.synchronize()
rows = [(ev.key, ev.self_device_time_total / 2e3) for ev in prof.key_averages() if ev.self_device_time_total > 0]
rows.sort(key=lambda r: -r[1])
print(json.dumps({"ms": round(statistics.median(ts), 2), "kernel_ms": round(sum(r[1] for r in rows), 2),
                  "top_kernels_ms": [[k[:70], round(v, 2)] for k, v in rows[:8]]}))
"""


def step(reps, warmup):
    if not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "py", "lib")):
        return "not measured: the reference Python is not staged under oracle/_ref/py"
    out = {}
    for mode in ("off", "on", "off", "on"):       # alternated, the last of each kept
        r = subprocess.run([sys.executable, "-c", STEP, mode, ROOT, str(reps), str(warmup)], capture_output=True,
                           text=True, cwd=ROOT)
        if r.returncode != 0:
            return f"failed ({mode}): {r.stderr[-400:]}"
        res = json.loads(r.stdout.strip().splitlines()[-1])
        out[f"deterministic_{mode}_ms"] = res["ms"]
        out[f"deterministic_{mode}_profile"] = {k: res[k] for k in ("kernel_ms", "top_kernels_ms")}
    out["ratio"] = round(out["deterministic_on_ms"] / out["deterministic_off_ms"], 3)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("determinism_bench: needs a CUDA device (a CPU run measures nothing)")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    res = {"bench": "determinism", "gpu": torch.cuda.get_device_name(dev), "power_limit_and_max_sm_clock": smi or "unknown",
           "grads": grads(dev, args.reps, args.warmup), "psp": psp(dev, args.reps, args.warmup),
           "step_b2": step(max(3, args.reps // 4), args.warmup)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
