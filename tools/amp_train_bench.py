"""What mixed precision buys in PVN3D training: prints ONE JSON line.

  * ops: the PointNet++ grouping / interpolation ops and the PSPNet backward at the training shapes (24 frames x 12288
    points, device FPS / ball query / three_nn plans; the PSP shapes of tools/determinism_bench.py), each in float32,
    natively in bf16 and fp16 (the pvn3d_*_16 entry points), and as the upcast composition the 16-bit forms replace
    (x.float(), the float32 op, .to(dtype)).  Grads and the PSP backward are timed with deterministic mode off
    ("atomic": the atomic entry points, torch's own PSP backward) and on ("ordered").  Each entry also gives the bytes
    the float32 and the 16-bit op must move (MB).
  * step: one training step (forward, model_fn's three losses, backward, an SGD step at lr 0) of the staged reference
    PVN3D (resnet34, pretrained=False, 480 x 640, N = 12288) at B = 2 and at the largest B in {24, 16, 8} whose float32
    step fits on the card (predicted from the float32 steps at B = 2 and 8, leaving 40 % of the card free): float32 (TF32 as torch
    defaults), bf16 autocast, fp16 autocast with GradScaler, each with deterministic mode off and on
    (compat.install(patch_deterministic=True), CUBLAS_WORKSPACE_CONFIG=:4096:8).  Step time
    (CUDA-event median) and peak allocated memory; at the largest B a torch.profiler table of the eight largest kernels
    of each precision (mode off), taken in a separate pass after the timed steps.  "not measured" when the reference
    Python is not staged under oracle/_ref/py.

Times are CUDA-event medians of `--reps` calls after `--warmup`, in milliseconds.

    python tools/amp_train_bench.py [--reps 20] [--warmup 3]
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

from pvn3d_b200 import _ext, deterministic, synth  # noqa: E402

B, N = 24, 12288
SA_LEVELS = [(12288, 2048, (0.0175, 0.025), (16, 32)), (2048, 1024, (0.025, 0.05), (16, 32)),
             (1024, 512, (0.05, 0.1), (16, 32)), (512, 128, (0.1, 0.2), (16, 32))]
SA_C = (6, 96, 256, 512)
FP_C = (256, 512, 512, 1024)
DT = {"bf16": torch.bfloat16, "fp16": torch.float16}


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


def forms(make, reps, warmup):
    """{float32, bf16, fp16, bf16_upcast, fp16_upcast: ms}; make(dtype, upcast) -> the call to time"""
    res = {"fp32": timed(make(torch.float32, False), reps, warmup)}
    for name, dt in DT.items():
        res[name] = timed(make(dt, False), reps, warmup)
        res[name + "_upcast"] = timed(make(dt, True), reps, warmup)
    return res


def modes(make, reps, warmup):
    out = {"atomic": forms(make, reps, warmup)}
    torch.use_deterministic_algorithms(True)
    try:
        out["ordered"] = forms(make, reps, warmup)
    finally:
        torch.use_deterministic_algorithms(False)
    return out


def _up(fn, dt):
    """the upcast composition: widen the 16-bit operand, run the float32 op, round the result"""
    return lambda x, *rest: fn(x.float(), *rest).to(dt)


def ops(dev, reps, warmup):
    frames = synth.make_batch("ycb", B, n_points=N, config_id=31)
    xyz = torch.from_numpy(np.stack([f.pcld for f in frames])).to(dev).contiguous()
    levels = [xyz]
    for _, m, _, _ in SA_LEVELS:
        levels.append(_ext.gather_xyz(levels[-1], _ext.furthest_point_sampling(levels[-1], m)))
    gen = torch.Generator(device=dev).manual_seed(0)
    res = {}

    def call(fn, x, args, dt, upcast):
        xs = x.to(dt)
        f = _up(fn, dt) if upcast else fn
        return lambda: f(xs, *args)

    for li, (n, m, radii, nss) in enumerate(SA_LEVELS):
        for r, ns in zip(radii, nss):
            idx = _ext.ball_query(levels[li + 1], levels[li], r, ns)
            feats = torch.randn((B, SA_C[li], n), generator=gen, device=dev)
            g = torch.randn((B, SA_C[li], m, ns), generator=gen, device=dev)
            mb = lambda e: round((B * SA_C[li] * (n + m * ns) * e + idx.numel() * 4) / 1e6, 1)   # noqa: E731
            res[f"group_fwd_SA{li + 1}_ns{ns}"] = {
                **forms(lambda dt, up: call(_ext.group_points, feats, (idx,), dt, up), reps, warmup),
                "mb_fp32": mb(4), "mb_16": mb(2)}
            res[f"group_grad_SA{li + 1}_ns{ns}"] = {
                **modes(lambda dt, up: call(_ext.group_points_grad, g, (idx, n), dt, up), reps, warmup),
                "mb_fp32": mb(4), "mb_16": mb(2)}
    for lu in range(4):
        d2, idx = _ext.three_nn(levels[lu], levels[lu + 1])
        recip = 1.0 / (torch.sqrt(d2) + 1e-8)
        w = (recip / recip.sum(2, keepdim=True)).contiguous()
        n, m = levels[lu].size(1), levels[lu + 1].size(1)
        feats = torch.randn((B, FP_C[lu], m), generator=gen, device=dev)
        g = torch.randn((B, FP_C[lu], n), generator=gen, device=dev)
        mb = lambda e: round((B * FP_C[lu] * (n + m) * e + idx.numel() * 8) / 1e6, 1)   # noqa: E731
        res[f"interp_fwd_FP{lu + 1}"] = {
            **forms(lambda dt, up: call(_ext.three_interpolate, feats, (idx, w), dt, up), reps, warmup),
            "mb_fp32": mb(4), "mb_16": mb(2)}
        res[f"interp_grad_FP{lu + 1}"] = {
            **modes(lambda dt, up: call(_ext.three_interpolate_grad, g, (idx, w, m), dt, up), reps, warmup),
            "mb_fp32": mb(4), "mb_16": mb(2)}
    return res


def psp(dev, reps, warmup):
    """the backward alone (torch.autograd.grad of a retained graph); the upcast form runs the op on x.float() and
    rounds the input gradient"""
    gen = torch.Generator(device=dev).manual_seed(1)
    res = {}

    def case(name, x_shape, fwd):
        x32 = torch.randn(x_shape, generator=gen, device=dev)
        g32 = None

        def make(dt, upcast):
            nonlocal g32
            if dt == torch.float32 or upcast:
                x = x32.clone().requires_grad_(True)
                y = fwd(x)
            else:
                x = x32.to(dt).requires_grad_(True)
                y = fwd(x)
            if g32 is None:
                g32 = torch.randn(y.shape, generator=gen, device=dev)
            g = g32 if dt == torch.float32 else g32.to(dt)
            if upcast:
                return lambda: torch.autograd.grad(y, x, g.float(), retain_graph=True)[0].to(dt)
            return lambda: torch.autograd.grad(y, x, g, retain_graph=True)
        res[name] = modes(make, reps, warmup)

    for s in (2, 3, 6):
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
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
from helpers import load_reference_python
from pvn3d_b200 import compat
assert load_reference_python() is not None
compat.install(patch_deterministic=True)
import lib.pvn3d as P
from lib.loss import FocalLoss, OFLoss
from lib.pspnet import Modified_PSPNet
P.modified_psp_models["resnet34"] = lambda: Modified_PSPNet(sizes=(1, 2, 3, 6), psp_size=512, deep_features_size=256,
                                                            backend="resnet34", pretrained=False)
dev = torch.device("cuda:0")
torch.manual_seed(0)
model = P.PVN3D(num_classes=22, pcld_input_channels=6, pcld_use_xyz=True, num_kps=8, num_points=12288).to(dev).train()
opt = torch.optim.SGD(model.parameters(), lr=0.0)
crit, crit_of = FocalLoss(gamma=2), OFLoss()
n = 12288
reps, warmup = int(sys.argv[3]), int(sys.argv[4])
DT = {"fp32": None, "bf16": torch.bfloat16, "fp16": torch.float16}

def inputs(b):
    gen = torch.Generator().manual_seed(1)
    return dict(rgb=torch.rand((b, 3, 480, 640), generator=gen).to(dev),
                cld=torch.randn((b, n, 9), generator=gen).to(dev) * 0.1,
                choose=torch.stack([torch.randperm(480 * 640, generator=gen)[:n] for _ in range(b)])[:, None].to(dev),
                labels=torch.randint(0, 22, (b, n), generator=gen).to(dev),
                kp=torch.randn((b, n, 8, 3), generator=gen).to(dev) * 0.05,
                ctr=torch.randn((b, n, 1, 3), generator=gen).to(dev) * 0.05)

def make_step(x, prec):
    scaler = torch.amp.GradScaler("cuda", enabled=prec == "fp16")
    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=DT[prec], enabled=DT[prec] is not None):
            pk, ps, pc = model(x["cld"], x["rgb"], x["choose"])
            loss = crit(ps.view(x["labels"].numel(), -1), x["labels"].view(-1)).sum() * 2.0 \
                + crit_of(pk, x["kp"], x["labels"]).sum() + crit_of(pc, x["ctr"], x["labels"]).sum()
        scaler.scale(loss).backward()
        scaler.step(opt)
        scaler.update()
    return step

def measure(step):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    ts = []
    for _ in range(reps):
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); step(); e.record(); e.synchronize()
        ts.append(a.elapsed_time(e))
    return {"ms": round(statistics.median(ts), 2), "peak_gib": round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2)}

def fp32_peak(b):
    x = inputs(b)
    step = make_step(x, "fp32")
    step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    step()
    torch.cuda.synchronize()
    free, total = torch.cuda.mem_get_info(dev)
    return x, torch.cuda.max_memory_allocated(dev), total - free

if sys.argv[2] == "max":
    # the largest B in {24, 16, 8} whose float32 step fits, predicted from B = 2 and 8: the allocated peak grows
    # linearly in B, on top of what the device already holds at B = 8 (caching allocator, cuDNN / cuBLAS workspaces),
    # and 40 % of the card is left free for the other precisions' workspaces.  Nothing runs at a B predicted not to fit.
    _, p2, _ = fp32_peak(2)
    x, p8, used8 = fp32_peak(8)
    per_frame = (p8 - p2) / 6
    cap = 0.6 * torch.cuda.get_device_properties(dev).total_memory
    b = max([c for c in (8, 16, 24) if used8 + (c - 8) * per_frame <= cap])
    x = x if b == 8 else inputs(b)
    fit = {"peak_gib_b2": round(p2 / 2 ** 30, 2), "peak_gib_b8": round(p8 / 2 ** 30, 2),
           "device_used_gib_b8": round(used8 / 2 ** 30, 2)}
else:
    b = int(sys.argv[2])
    x = inputs(b)
    fit = {}
res = {"b": b, **fit}
for det in (False, True):
    torch.use_deterministic_algorithms(det)
    for prec in ("fp32", "bf16", "fp16"):
        try:
            res[f"{prec}_det_{'on' if det else 'off'}"] = measure(make_step(x, prec))
        except RuntimeError as e:
            res[f"{prec}_det_{'on' if det else 'off'}"] = {"raised": str(e)[:300]}
            torch.cuda.empty_cache()
torch.use_deterministic_algorithms(False)
if sys.argv[2] == "max":
    from torch.profiler import ProfilerActivity, profile
    prof_res = {}
    for prec in ("fp32", "bf16", "fp16"):
        step = make_step(x, prec)
        step()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(2):
                step()
            torch.cuda.synchronize()
        rows = [(ev.key, ev.self_device_time_total / 2e3) for ev in prof.key_averages() if ev.self_device_time_total > 0]
        rows.sort(key=lambda r: -r[1])
        prof_res[prec] = {"kernel_ms": round(sum(r[1] for r in rows), 2),
                          "top_kernels_ms": [[k[:70], round(v, 2)] for k, v in rows[:8]]}
    res["profile_det_off"] = prof_res
print(json.dumps(res))
"""


def step(which, reps, warmup):
    if not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "py", "lib")):
        return "not measured: the reference Python is not staged under oracle/_ref/py"
    r = subprocess.run([sys.executable, "-c", STEP, ROOT, which, str(reps), str(warmup)], capture_output=True, text=True,
                       cwd=ROOT)
    if r.returncode != 0:
        return f"failed (B {which}): {r.stderr[-600:]}"
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("amp_train_bench: needs a CUDA device (a CPU run measures nothing)")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    res = {"bench": "amp_train", "gpu": torch.cuda.get_device_name(dev), "power_limit_and_max_sm_clock": smi or "unknown",
           "ops": ops(dev, args.reps, args.warmup), "psp": psp(dev, args.reps, args.warmup)}
    steps = max(3, args.reps // 4)
    res["step"] = {"b2": step("2", steps, args.warmup), "bmax": step("max", steps, args.warmup)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
