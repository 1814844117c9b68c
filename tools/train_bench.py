"""Time the training-side GPU paths of pvn3d_b200.train_utils and print ONE JSON line (with the GPU's name and power
limit, read in the same run):

  loss_ycb / loss_lm   forward + backward of model_fn's three loss terms at B=24, N=12288 (YCB: C=22, K=8; LineMOD:
                       C=2, K=8): PVN3DLoss (two forward launches, one backward launch) against the reference's
                       lib/loss.py FocalLoss(gamma=2) + 2x OFLoss when the reference Python is staged (oracle/_ref/py),
                       otherwise against a float32 torch restatement of the same code (baseline="torch_restated")
  targets              TrainTargets.compute at B=24, N=12288, 22 slots, K=8
  train_batch          train_batch for 24 YCB-shape frames (synth.make_icp_depth_batch) with fill="multiscale", stage
                       by stage: the depth fill, the rest of FrameInputBuilder.build, the targets, and the whole call

Times are medians of CUDA-event-timed calls after warm-up, in microseconds (host launch overhead included: the small
calls are launch-bound); *kernel* entries are the device time of the library's own kernels from torch.profiler.

    python tools/train_bench.py [--reps 20] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from pvn3d_b200 import synth  # noqa: E402
from pvn3d_b200 import train_utils as T  # noqa: E402
from pvn3d_b200.frame_input import FrameInputBuilder  # noqa: E402

B, N = 24, 12288


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, watts = (s.strip() for s in out.splitlines()[0].split(","))
        return name, float(watts)
    except Exception:  # noqa: BLE001 -- reported as unknown
        return torch.cuda.get_device_name(0), None


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
        ts.append(a.elapsed_time(b) * 1e3)
    return round(float(np.median(ts)), 1)


def kernel_us(fn, names):
    """device time (us) of the kernels whose name contains one of `names` in one call of fn (torch.profiler)"""
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = 0.0
    for e in prof.key_averages():
        if any(n in e.key for n in names):
            tot += getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0.0)
    return round(float(tot), 1)


class _TorchFocal(torch.nn.Module):
    """lib/loss.py's FocalLoss forward, restated in float32 torch (alpha None)"""

    def __init__(self, gamma):
        super().__init__()
        self.gamma = gamma

    def forward(self, x, t):
        logpt = torch.log_softmax(x, 1).gather(1, t.view(-1, 1)).view(-1)
        pt = logpt.detach().exp()
        return (-1 * (1 - pt) ** self.gamma * logpt).mean()


class _TorchOF(torch.nn.Module):
    """lib/loss.py's of_l1_loss, restated in float32 torch"""

    def forward(self, pred, targ, labels):
        w = (labels > 1e-8).float()
        bs, k, n, c = pred.size()
        w = w.view(bs, 1, n, 1).repeat(1, k, 1, 1).contiguous()
        targ = targ.view(bs, n, k, 3).permute(0, 2, 1, 3).contiguous()
        d = w * torch.abs(pred - targ)
        return torch.sum(d.view(bs, k, -1), 2) / (torch.sum(w.view(bs, k, -1), 2) + 1e-3)


def baseline_losses():
    from helpers import load_reference_python

    if load_reference_python() is not None:
        import importlib

        lib_loss = importlib.import_module("lib.loss")
        return "reference_lib_loss", lib_loss.FocalLoss(gamma=2), lib_loss.OFLoss()
    return "torch_restated", _TorchFocal(2), _TorchOF()


def bench_loss(c, reps, warmup, base):
    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(0)
    seg = (torch.randn(B, N, c, generator=g) * 3).to(dev).requires_grad_(True)
    labels = (torch.randint(0, c, (B, N), generator=g) * (torch.rand(B, N, generator=g) < 0.3)).to(dev)
    kp = (torch.randn(B, 8, N, 3, generator=g) * 0.1).to(dev).requires_grad_(True)
    ctr = (torch.randn(B, 1, N, 3, generator=g) * 0.1).to(dev).requires_grad_(True)
    kt = (torch.randn(B, N, 8, 3, generator=g) * 0.1).to(dev)
    ct = (torch.randn(B, N, 3, generator=g) * 0.1).to(dev)
    crit = T.PVN3DLoss()
    name, focal, of = base

    def ours():
        loss, _, _ = crit(kp, seg, ctr, kt, ct, labels)
        loss.backward()

    def ours_fwd():
        with torch.no_grad():
            crit(kp, seg, ctr, kt, ct, labels)

    def theirs():
        loss = focal(seg.view(labels.numel(), -1), labels.view(-1)).sum() * 2 + of(kp, kt, labels).sum() + \
            of(ctr, ct, labels).sum()
        _, cls = torch.max(seg, -1)
        (cls == labels).float().sum() / labels.numel()
        loss.backward()

    return {"fused_fwd_bwd_us": timed(ours, reps, warmup), "fused_fwd_us": timed(ours_fwd, reps, warmup),
            f"{name}_fwd_bwd_us": timed(theirs, reps, warmup),
            "fused_kernels_fwd_us": kernel_us(ours_fwd, ("train_loss_partials", "train_loss_finish")),
            "fused_kernels_bwd_us": kernel_us(ours, ("train_loss_backward",))}


def bench_targets(reps, warmup):
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(1)
    pcld = torch.from_numpy(rng.normal(0, 0.3, (B, N, 3)).astype(np.float32)).to(dev)
    labels = torch.from_numpy(rng.integers(0, 22, (B, N)).astype(np.int32)).to(dev)
    ids = torch.from_numpy(np.tile(np.r_[np.arange(1, 7), np.zeros(16)].astype(np.int32), (B, 1))).to(dev)
    rts = torch.from_numpy(rng.normal(0, 1, (B, 22, 3, 4))).to(dev)
    tt = T.TrainTargets(device=dev)
    fn = lambda: tt.compute(pcld, labels, ids, rts)  # noqa: E731
    return {"compute_us": timed(fn, reps, warmup), "kernel_us": kernel_us(fn, ("train_targets",))}


def bench_train_batch(reps, warmup):
    dev = torch.device("cuda:0")
    d = synth.make_icp_depth_batch(B, seed=3)
    depth, K, cs = (torch.from_numpy(d[k]).to(dev) for k in ("depth", "K", "cam_scale"))
    label = torch.from_numpy(d["label"]).to(dev)
    rgb = torch.from_numpy(np.random.default_rng(3).integers(0, 256, (B, 3, synth.H, synth.W), dtype=np.uint8)).to(dev)
    ids = torch.from_numpy((np.arange(22)[None] * d["present"]).astype(np.int64)).to(dev)
    rts = torch.from_numpy(d["gt"]).to(dev)
    builder = FrameInputBuilder(B, N, fill="multiscale", device=dev)
    plain = FrameInputBuilder(B, N, device=dev)
    tt = T.TrainTargets(device=dev)
    out = plain.build(depth, K, cs, rgb, 0, label_image=label)
    return {"depth_fill_us": timed(lambda: builder.filler.fill(depth, cs), reps, warmup),
            "build_without_fill_us": timed(lambda: plain.build(depth, K, cs, rgb, 0, label_image=label), reps, warmup),
            "targets_us": timed(lambda: tt.compute(out[3], out[5], ids, rts), reps, warmup),
            "train_batch_us": timed(lambda: T.train_batch(builder, tt, depth, K, cs, rgb, label, ids, rts, 0), reps,
                                    warmup)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    name, watts = gpu_info()
    base = baseline_losses()
    out = {"gpu": name, "power_limit_w": watts, "batch": B, "n_points": N, "baseline": base[0],
           "loss_ycb": bench_loss(22, a.reps, a.warmup, base), "loss_lm": bench_loss(2, a.reps, a.warmup, base),
           "targets": bench_targets(a.reps, a.warmup), "train_batch_ycb": bench_train_batch(a.reps, a.warmup)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
