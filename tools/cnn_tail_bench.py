"""Dense against sampled CNN tail (pvn3d_psp_tail_rows), timed on the device: ONE JSON line.

    python tools/cnn_tail_bench.py [--calls 5] [--rounds 3]

At 480 x 640 with N = 12288 sampled pixels, LineMOD batch 32 and YCB batch 16, on a seeded CNN with the reference's
layout (testing.StandInPSPNet: the real up_3 / final / final_seg modules):
  * tail alone, on a precomputed up_2 output: dense = up_3 + final + final_seg + pvn3d_gather_pixel_rows, as
    Modified_PSPNet.forward and FusedPVN3D run them; sampled = channels-last copy + pvn3d_psp_tail_rows; and the kernel
    alone on a channels-last map, with its FLOP and bytes computed from the shapes;
  * the whole CNN, dense against trunk + sampled tail, on the reference's own Modified_PSPNet(resnet34, pretrained=False)
    where the reference Python is staged under oracle/_ref/py ("not measured" otherwise);
  * torch.cuda.max_memory_allocated() of one call each way, and the difference of the two row sets over their scale.
Dense and sampled alternate `rounds` times in one process; each figure is the median of rounds * calls CUDA-event timings
after two warm-up calls per round.  cuDNN runs with torch's default allow_tf32 = True, the reference's setting.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pvn3d_b200 import compat, network, testing  # noqa: E402
from pvn3d_b200._lib import call, ptr  # noqa: E402
from pvn3d_b200.cnn_tail import PspTail  # noqa: E402
from pvn3d_b200.mlp import _layer_struct  # noqa: E402

H, W, N = 480, 640, 12288
SHAPES = (("linemod", 32), ("ycb", 16))
TF32_PEAK, HBM_PEAK = 495e12, 3.35e12     # H100 SXM data sheet, dense TF32 FLOP/s and HBM3 bytes/s (a 700 W card)


def timed(fn, calls):
    out = []
    for i in range(2 + calls):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        if i >= 2:
            out.append(e0.elapsed_time(e1))
    return out


def alternate(variants, rounds, calls):
    """{name: median ms} of the variants, run in turn `rounds` times"""
    ms = {k: [] for k in variants}
    for _ in range(rounds):
        for k, fn in variants.items():
            ms[k] += timed(fn, calls)
    return {k: round(statistics.median(v), 4) for k, v in ms.items()}


def peak_bytes(fn):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def kernel_model(b):
    """FLOP and bytes of one pvn3d_psp_tail_rows launch, from the shapes"""
    rows = b * N
    flop = rows * (576 * 64 + 64 * 128) * 2
    hbm = b * (H // 2) * (W // 2) * 64 * 4 + rows * (128 * 4 + 8)       # the map once, the rows, choose
    gathered = rows * 9 * 4 * 256 + (rows // 128) * 576 * 64 * 4         # what the SMs request: taps and the W1 stream
    return flop, hbm, gathered


def tail_alone(dev, b, rounds, calls):
    cnn = testing.StandInPSPNet(seed=0).to(dev)
    tail = PspTail.from_cnn(cnn)
    x_half = torch.randn(b, 64, H // 2, W // 2, device=dev, generator=torch.Generator(dev).manual_seed(b))
    choose = testing.sample_choose(b, N, H * W, seed=b).to(dev)
    t_dense = torch.empty(b * N, 128, device=dev)
    t_sampled = torch.empty(b * N, 128, device=dev)
    x_cl = x_half.permute(0, 2, 3, 1).contiguous()
    l1, l2 = _layer_struct(tail.layer1), _layer_struct(tail.layer2)

    def dense():
        p = cnn.up_3(x_half)
        emb, seg = cnn.final(p), cnn.final_seg(p).permute(0, 2, 3, 1).contiguous()
        network.gather_pixel_rows(emb.contiguous(), choose, t_dense)
        return seg

    def sampled():
        tail.rows(x_half, choose, t_sampled)

    def kernel():
        call("pvn3d_psp_tail_rows", dev, ptr(x_cl), b, H // 2, W // 2, ptr(choose), N, ctypes.addressof(l1),
             ctypes.addressof(l2), ptr(tail.slope), 0, ptr(t_sampled), 128, 0)

    ms = alternate({"dense_ms": dense, "sampled_ms": sampled, "kernel_ms": kernel}, rounds, calls)
    flop, hbm, gathered = kernel_model(b)
    t = ms["kernel_ms"] * 1e-3
    bounds = {"tf32_peak_ms": round(flop / TF32_PEAK * 1e3, 4), "hbm_peak_ms": round(hbm / HBM_PEAK * 1e3, 4)}
    scale = float(t_dense.abs().max())
    err = (t_sampled - t_dense).abs()
    return {**ms, "speedup": round(ms["dense_ms"] / ms["sampled_ms"], 2),
            "kernel": {"gflop": round(flop / 1e9, 2), "hbm_mb": round(hbm / 1e6, 1), "gathered_mb": round(gathered / 1e6, 1),
                       "tflops": round(flop / t / 1e12, 2), "gathered_tb_s": round(gathered / t / 1e12, 3), **bounds,
                       "nearer_bound": max(bounds, key=bounds.get)},
            "peak_bytes": {"dense": peak_bytes(dense), "sampled": peak_bytes(sampled)},
            "rows_diff_over_scale": {"max": float(err.max()) / scale, "mean": float(err.mean()) / scale}}


def whole_cnn(dev, b, rounds, calls):
    root = os.path.join(ROOT, "oracle", "_ref", "py")
    if not os.path.isdir(os.path.join(root, "lib")):
        return "not measured: the reference Python is not staged under oracle/_ref/py"
    compat.install(root)
    from lib.pspnet import Modified_PSPNet

    torch.manual_seed(0)
    cnn = Modified_PSPNet(sizes=(1, 2, 3, 6), psp_size=512, deep_features_size=256, backend="resnet34", pretrained=False)
    cnn = testing.randomize_bn_(cnn).to(dev).eval()
    tail = PspTail.from_cnn(cnn)
    rgb = torch.rand(b, 3, H, W, device=dev, generator=torch.Generator(dev).manual_seed(b))
    choose = testing.sample_choose(b, N, H * W, seed=b).to(dev)
    t_dense = torch.empty(b * N, 128, device=dev)
    t_sampled = torch.empty(b * N, 128, device=dev)

    def dense():
        emb, _ = cnn(rgb)
        network.gather_pixel_rows(emb.contiguous(), choose, t_dense)

    def sampled():
        tail.rows(tail.trunk(rgb), choose, t_sampled)

    ms = alternate({"dense_ms": dense, "sampled_ms": sampled}, rounds, calls)
    scale = float(t_dense.abs().max())
    err = (t_sampled - t_dense).abs()
    return {**ms, "speedup": round(ms["dense_ms"] / ms["sampled_ms"], 2),
            "peak_bytes": {"dense": peak_bytes(dense), "sampled": peak_bytes(sampled)},
            "rows_diff_over_scale": {"max": float(err.max()) / scale, "mean": float(err.mean()) / scale}}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--calls", type=int, default=5, help="timed calls per variant and round (>= 5)")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cnn_tail_bench: needs a CUDA device (a CPU run measures nothing)")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    res = {"bench": "cnn_tail", "gpu": torch.cuda.get_device_name(dev), "power_limit_and_max_sm_clock": smi or "unknown",
           "image": [H, W], "points": N, "calls": args.calls * args.rounds, "cudnn_allow_tf32": torch.backends.cudnn.allow_tf32}
    with torch.no_grad():
        for name, b in SHAPES:
            res[name] = {"batch": b, "tail": tail_alone(dev, b, args.rounds, max(5, args.calls)),
                         "whole_cnn": whole_cnn(dev, b, args.rounds, max(5, args.calls))}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
