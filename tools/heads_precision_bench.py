"""Time the heads and the network forward at precision "tf32" against "bf16" and print ONE JSON line.

Per batch, at 12288 points, LineMOD shape (batch 32) and YCB shape (batch 16):
  heads    FusedHeads(precision=...) on fixed random [B,128,N] embeddings;
  network  FusedPVN3D(precision=...) with the FixedEmbedding CNN stand-in of tools/network_bench.py (the CNN is excluded).
Each pair alternates three times in one process; each entry is the median of --reps calls timed with CUDA events after
--warmup calls.  Also reported, per config:
  * the deviation of the bf16 outputs from the tf32 ones: mean and max |bf16 - tf32| over the mean |tf32| of each output;
  * "computed_from_shapes": the FLOPs the heads' launches execute (padded shapes) and the activation bytes they read and
    write, per batch -- arithmetic, not measurements;
  * "achieved": those FLOPs and bytes over the measured median heads time, next to the H100 SXM data-sheet peaks (dense
    TF32 494.7 and BF16 989.4 TFLOP/s, HBM3 3.35 TB/s).
The GPU name and power limit are read in the same run.  Not part of bench.py.

    python tools/heads_precision_bench.py [--reps 5] [--warmup 2]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from network_bench import CONFIGS, IMG_H, IMG_W, N_POINTS, FixedEmbedding, power_limit_w, timed  # noqa: E402
from pvn3d_b200 import synth, testing  # noqa: E402
from pvn3d_b200.heads import FusedHeads  # noqa: E402
from pvn3d_b200.network import FusedPVN3D  # noqa: E402

DATASHEET = {"tf32_dense_tflops": 494.7, "bf16_dense_tflops": 989.4, "hbm3_tb_per_s": 3.35}


def heads_work(h: FusedHeads, rows: int):
    """(FLOPs, activation bytes) of one FusedHeads.run over `rows` points, from the packed shapes (n % 128 == 0 path)"""
    es = 2 if h.precision == "bf16" else 4
    launches = [(256, h.la, es), (512, h.lb, 0)]                      # (a_cols, layer, bytes per stored element)
    for hd in h.heads:
        launches.append((768, hd.first, es))
        for i, pl in enumerate(hd.rest):
            launches.append((pl.k_pad, pl, 4 if i == len(hd.rest) - 1 else es))
    flops = sum(2 * rows * pl.k_pad * pl.n_pad for _, pl, _ in launches)
    act_bytes = sum(rows * a_cols * es + rows * pl.n_pad * out_es for a_cols, pl, out_es in launches)
    return flops, act_bytes


def deviation(got, ref):
    out = {}
    for name, g, r in zip(("kp_of", "seg", "ctr_of"), got, ref):
        scale = float(r.abs().mean())
        d = (g - r).abs()
        out[name] = {"mean": float(d.mean()) / scale, "max": float(d.max()) / scale}
    return out


def alternate(fns, reps, warmup):
    ms = {k: [] for k in fns}
    for _ in range(3):
        for k, fn in fns.items():
            ms[k].append(round(timed(fn, reps, warmup), 3))
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    res = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "n_points": N_POINTS,
           "reps": args.reps, "warmup": args.warmup, "datasheet_h100_sxm": DATASHEET, "configs": {}}
    for shape, b in CONFIGS:
        g = torch.Generator(device=dev).manual_seed(b)
        model = testing.StandInPVN3D(N_POINTS, seed=5)
        model.cnn = FixedEmbedding(torch.randn(b, 128, IMG_H, IMG_W, generator=g, device=dev).relu())
        model = model.to(dev).eval()
        frames = synth.make_batch(shape, b, n_points=N_POINTS, config_id=2, lm_obj_id=1 if shape == "linemod" else None)
        pc = torch.from_numpy(np.stack([f.cld_rgb_nrm for f in frames])).to(dev).contiguous()
        rgb = torch.zeros(b, 3, 1, 1, device=dev)
        choose = testing.sample_choose(b, N_POINTS, IMG_H * IMG_W, seed=b).to(dev)
        rgb_emb = torch.randn(b, 128, N_POINTS, generator=g, device=dev)
        cld_emb = torch.randn(b, 128, N_POINTS, generator=g, device=dev).relu()
        mods = (model.rgbd_feat, model.SEG_layer, model.KpOF_layer, model.CtrOf_layer)
        hd = {p: FusedHeads(*mods, dev, precision=p) for p in ("tf32", "bf16")}
        net = {p: FusedPVN3D(model, dev, precision=p) for p in ("tf32", "bf16")}
        with torch.no_grad():
            heads_ms = alternate({p: (lambda p=p: hd[p](rgb_emb, cld_emb)) for p in hd}, args.reps, args.warmup)
            net_ms = alternate({p: (lambda p=p: net[p](pc, rgb, choose)) for p in net}, args.reps, args.warmup)
            heads_dev = deviation(hd["bf16"](rgb_emb, cld_emb), hd["tf32"](rgb_emb, cld_emb))
            net_dev = deviation(net["bf16"](pc, rgb, choose), net["tf32"](pc, rgb, choose))
        cfg = {"heads_ms": heads_ms, "network_ms": net_ms,
               "heads_bf16_speedup_of_medians": round(float(np.median(heads_ms["tf32"]) / np.median(heads_ms["bf16"])), 3),
               "network_bf16_speedup_of_medians": round(float(np.median(net_ms["tf32"]) / np.median(net_ms["bf16"])), 3),
               "bf16_vs_tf32_deviation_over_output_scale": {"heads": heads_dev, "network": net_dev},
               "computed_from_shapes": {}, "achieved": {}}
        for p in ("tf32", "bf16"):
            flops, nbytes = heads_work(hd[p], b * N_POINTS)
            t = float(np.median(heads_ms[p])) * 1e-3
            cfg["computed_from_shapes"][p] = {"heads_gflop_per_batch": round(flops / 1e9, 1),
                                              "heads_activation_gb_per_batch": round(nbytes / 1e9, 2)}
            cfg["achieved"][p] = {"heads_tflops": round(flops / t / 1e12, 1), "heads_activation_tb_per_s": round(nbytes / t / 1e12, 2)}
        res["configs"][f"{shape}_b{b}"] = cfg
        del model, hd, net
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
