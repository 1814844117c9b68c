"""Time the PVN3D network forward without its CNN and print ONE JSON line.

Per batch, at 12288 points, LineMOD shape (batch 32) and YCB shape (batch 16):
  (a) the hand composition of the two engines: torch.gather of the embedding, FusedPointnet2MSG, FusedHeads;
  (b) FusedPVN3D (the gather and FP1 write the heads' activation table directly);
  (c) the reference's module-graph PVN3D.forward on this package's _ext with TF32 on, where oracle/_ref/py is staged
      ("unavailable" otherwise).
All three use a stand-in CNN that returns one precomputed random [B,128,480,640] embedding, so the CNN is in none of
them.  Weights: pvn3d_b200.testing.StandInPVN3D.  (a) and (b) alternate three times in the same process; each entry
is the median of --reps calls timed with CUDA events after --warmup calls.  Whether (a) and (b) give the same bits is
reported per config.  Not part of bench.py.

    python tools/network_bench.py [--reps 5] [--warmup 2]
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
from pvn3d_b200 import synth, testing  # noqa: E402
from pvn3d_b200.heads import FusedHeads  # noqa: E402
from pvn3d_b200.mlp import FusedPointnet2MSG  # noqa: E402
from pvn3d_b200.network import FusedPVN3D  # noqa: E402

N_POINTS, IMG_H, IMG_W = 12288, 480, 640
CONFIGS = (("linemod", 32), ("ycb", 16))


class FixedEmbedding(torch.nn.Module):
    """a CNN stand-in: returns the same precomputed embedding for any rgb"""

    def __init__(self, emb):
        super().__init__()
        self.emb = emb

    def forward(self, rgb):
        return self.emb, None


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:  # noqa: BLE001 -- reported as unknown
        return None


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


def reference_forward(model, dev):
    """(c): the reference's PVN3D.forward on reference modules with the same weights, or None if not staged"""
    if not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "py", "lib")):
        return None
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from helpers import load_reference_python
    from make_golden_network import reference_pvn3d

    ref = load_reference_python()
    if ref is None:
        return None
    rm = reference_pvn3d(ref, model, N_POINTS).to(dev)
    rm.cnn = model.cnn
    return lambda *x: ref.pvn3d.PVN3D.forward(rm, *x)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = True
    res = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "n_points": N_POINTS,
           "image": [IMG_H, IMG_W], "reps": args.reps, "warmup": args.warmup, "configs": {}}
    for shape, b in CONFIGS:
        g = torch.Generator(device=dev).manual_seed(b)
        model = testing.StandInPVN3D(N_POINTS, seed=5)
        model.cnn = FixedEmbedding(torch.randn(b, 128, IMG_H, IMG_W, generator=g, device=dev))
        model = model.to(dev).eval()
        frames = synth.make_batch(shape, b, n_points=N_POINTS, config_id=2, lm_obj_id=1 if shape == "linemod" else None)
        pc = torch.from_numpy(np.stack([f.cld_rgb_nrm for f in frames])).to(dev).contiguous()
        rgb = torch.zeros(b, 3, 1, 1, device=dev)
        choose = testing.sample_choose(b, N_POINTS, IMG_H * IMG_W, seed=b).to(dev)
        pn2 = FusedPointnet2MSG(model.pointnet2, dev)
        heads = FusedHeads(model.rgbd_feat, model.SEG_layer, model.KpOF_layer, model.CtrOf_layer, dev)
        net = FusedPVN3D(model, dev)

        def hand():
            out_rgb, _ = model.cnn(rgb)
            rgb_emb = torch.gather(out_rgb.view(b, 128, -1), 2, choose.repeat(1, 128, 1))
            return heads(rgb_emb, pn2(pc))

        def fused():
            return net(pc, rgb, choose)

        with torch.no_grad():
            same = all(torch.equal(x, y) for x, y in zip(hand(), fused()))
            a_ms, b_ms = [], []
            for _ in range(3):
                a_ms.append(round(timed(hand, args.reps, args.warmup), 3))
                b_ms.append(round(timed(fused, args.reps, args.warmup), 3))
            ref = reference_forward(model, dev)
            c_ms = "unavailable" if ref is None else round(timed(lambda: ref(pc, rgb, choose), args.reps, args.warmup), 3)
        res["configs"][f"{shape}_b{b}"] = {"a_hand_ms": a_ms, "b_fused_ms": b_ms, "c_module_graph_ms": c_ms,
                                            "a_b_bit_identical": same}
        del model, pn2, heads, net, ref
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
