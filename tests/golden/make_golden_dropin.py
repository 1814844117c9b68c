"""Record what the UNMODIFIED reference computes in tests/test_reference_dropin_gpu.py and tests/test_heads_gpu.py
(weights and inputs from tests/helpers.py), so that those tests run without a reference checkout.  Needs a GPU and
oracle/_ref/{_ext.so,py}:  python tests/golden/make_golden_dropin.py OUT_DIR  -> OUT_DIR/{dropin,heads}_ref.npz
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import (HEADS_CASES, PN2MSG_POINTS, heads_inputs, heads_modules, heads_points,  # noqa: E402
                     load_ref_ext, load_reference_python, sa_feature_grad, sa_module_and_inputs)
from pvn3d_b200 import synth, testing  # noqa: E402


def reference_heads(ref, dev):
    import lib.utils.etw_pytorch_utils as pt_utils
    from torch import nn

    fusion = ref.pvn3d.DenseFusion(2048)
    # the three stacks exactly as PVN3D.__init__ builds them (pvn3d.py:245-267)
    seg = (pt_utils.Seq(1792).conv1d(1024, bn=True, activation=nn.ReLU()).conv1d(512, bn=True, activation=nn.ReLU())
           .conv1d(128, bn=True, activation=nn.ReLU()).conv1d(22, activation=None))
    kpof = (pt_utils.Seq(1792).conv1d(1024, bn=True, activation=nn.ReLU()).conv1d(512, bn=True, activation=nn.ReLU())
            .conv1d(256, bn=True, activation=nn.ReLU()).conv1d(8 * 3, activation=None))
    ctrof = (pt_utils.Seq(1792).conv1d(1024, bn=True, activation=nn.ReLU()).conv1d(512, bn=True, activation=nn.ReLU())
             .conv1d(128, bn=True, activation=nn.ReLU()).conv1d(3, activation=None))
    mods = [fusion, seg, kpof, ctrof]
    for m, src in zip(mods, heads_modules()):
        m.load_state_dict(src.state_dict(), strict=True)
    return [m.to(dev).eval() for m in mods]


def reference_heads_forward(mods, rgb_emb, cld_emb):
    fusion, seg, kpof, ctrof = mods
    bs, _, n = cld_emb.shape
    fusion.ap1 = torch.nn.AvgPool1d(n)                      # DenseFusion(num_points) pools over all points (:165)
    with torch.no_grad():
        f = fusion(rgb_emb, cld_emb)
        pred_rgbd_seg = seg(f).transpose(1, 2).contiguous()                              # pvn3d.py:297
        pred_kp_of = kpof(f).view(bs, 8, 3, n).permute(0, 1, 3, 2).contiguous()          # :298-302
        pred_ctr_of = ctrof(f).view(bs, 1, 3, n).permute(0, 1, 3, 2).contiguous()        # :303-306
    return pred_kp_of, pred_rgbd_seg, pred_ctr_of


def main(out_dir):
    ref, ref_ext = load_reference_python(), load_ref_ext()
    assert ref is not None and ref_ext is not None, "oracle/_ref not staged"
    dev = torch.device("cuda:0")
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    out = {}
    torch.manual_seed(0)
    model = ref.pvn3d.Pointnet2MSG(input_channels=6)
    testing.randomize_bn_(model, 1)
    model = model.to(dev).eval()
    frames = synth.make_batch("ycb", 2, n_points=12288, config_id=11)
    x = torch.from_numpy(np.stack([f.cld_rgb_nrm for f in frames])).to(dev)
    ref.pn2_utils._ext = ref_ext
    with torch.no_grad():
        y = model(x)
    out["pn2msg_y"] = y[..., torch.from_numpy(PN2MSG_POINTS).to(dev)].cpu().numpy()
    from lib.pointnet2_utils import pointnet2_modules as ref_mod

    mine, xyz, feat = sa_module_and_inputs()
    sa = ref_mod.PointnetSAModuleMSG(npoint=64, radii=[0.1, 0.2], nsamples=[8, 16], mlps=[[6, 16, 32], [6, 16, 32]])
    sa.load_state_dict(mine.state_dict(), strict=True)
    out["sa_grad"] = sa_feature_grad(sa.to(dev).eval(), xyz.to(dev), feat.to(dev)).cpu().numpy()
    for shape in ("ycb", "linemod"):
        f = synth.make_frame(shape, n_points=4096, seed=77, lm_obj_id=1 if shape == "linemod" else None)
        args = [torch.from_numpy(a).to(dev) for a in (f.pcld, f.labels, f.ctr_of, f.kp_of)]
        if shape == "ycb":
            ids, poses = ref.eval_utils.cal_frame_poses(*args, True, 22, True)
            out["ids_ycb"] = np.asarray(ids, np.int64)
        else:
            poses = ref.eval_utils.cal_frame_poses_lm(*args, True, 2, False, 1)
        out[f"poses_{shape}"] = np.stack([np.asarray(p, np.float64) for p in poses])
    os.makedirs(out_dir, exist_ok=True)
    np.savez_compressed(os.path.join(out_dir, "dropin_ref.npz"), **out)
    print({k: v.shape for k, v in out.items()})

    mods = reference_heads(ref, dev)
    hout = {}
    for b, n in HEADS_CASES:
        rgb, cld = heads_inputs(b, n)
        kp, seg, ctr = reference_heads_forward(mods, rgb.to(dev), cld.to(dev))
        pts = torch.from_numpy(heads_points(n)).to(dev)
        for name, full, sample in (("kp_of", kp, kp[:, :, pts]), ("seg", seg, seg[:, pts]), ("ctr_of", ctr, ctr[:, :, pts])):
            hout[f"{name}_{b}x{n}"] = sample.float().cpu().numpy()
            hout[f"{name}_{b}x{n}_scale"] = np.float64(full.abs().double().mean().item())
    np.savez_compressed(os.path.join(out_dir, "heads_ref.npz"), **hout)
    print({k: np.shape(v) for k, v in hout.items()})


if __name__ == "__main__":
    main(sys.argv[1])
