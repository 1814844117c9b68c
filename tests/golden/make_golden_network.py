"""Record what the reference's UNMODIFIED PVN3D.forward (pvn3d/lib/pvn3d.py:269-310) computes for the model and inputs
of tests/network_cases.py, so that tests/test_network_gpu.py compares FusedPVN3D with it without a reference checkout.

The reference PVN3D is created with PVN3D.__new__ + nn.Module.__init__ (its constructor builds ModifiedResnet, which
downloads a pretrained checkpoint): the CNN is the stand-in of the test, the PointNet++, DenseFusion and head modules
are the reference's own classes loaded with the test's weights.  fp32 (TF32 off), the reference's compiled _ext where
oracle/_ref/_ext.so exists.  Needs a GPU and oracle/_ref/py:
    python tests/golden/make_golden_network.py OUT_DIR  -> OUT_DIR/network_ref.npz
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import load_ref_ext, load_reference_python  # noqa: E402
from network_cases import NETWORK_CASES, network_inputs, network_model, network_points  # noqa: E402


def reference_pvn3d(ref, standin, n):
    import lib.utils.etw_pytorch_utils as pt_utils
    from torch import nn

    def seq(widths, out):
        s = pt_utils.Seq(1792)
        for w in widths:
            s = s.conv1d(w, bn=True, activation=nn.ReLU())
        return s.conv1d(out, activation=None)

    model = ref.pvn3d.PVN3D.__new__(ref.pvn3d.PVN3D)
    nn.Module.__init__(model)
    model.num_kps = standin.num_kps
    model.cnn = standin.cnn
    model.pointnet2 = ref.pvn3d.Pointnet2MSG(input_channels=6)
    model.rgbd_feat = ref.pvn3d.DenseFusion(n)
    model.SEG_layer = seq((1024, 512, 128), 22)
    model.KpOF_layer = seq((1024, 512, 256), standin.num_kps * 3)
    model.CtrOf_layer = seq((1024, 512, 128), 3)
    model.load_state_dict(standin.state_dict(), strict=True)
    return model.eval()


def main(out_dir):
    ref, ref_ext = load_reference_python(), load_ref_ext()
    assert ref is not None, "oracle/_ref/py not staged"
    if ref_ext is not None:
        ref.pn2_utils._ext = ref_ext
    print("PointNet++ ops:", "reference _ext" if ref_ext is not None else "pvn3d_b200._ext")
    dev = torch.device("cuda:0")
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    out = {}
    for b, n in NETWORK_CASES:
        model = reference_pvn3d(ref, network_model(n), n).to(dev)
        pc, rgb, choose = (t.to(dev) for t in network_inputs(b, n))
        with torch.no_grad():
            kp, seg, ctr = ref.pvn3d.PVN3D.forward(model, pc, rgb, choose)
        pts = torch.from_numpy(network_points(n)).to(dev)
        for name, full, sample in (("kp_of", kp, kp[:, :, pts]), ("seg", seg, seg[:, pts]), ("ctr_of", ctr, ctr[:, :, pts])):
            out[f"{name}_{b}x{n}"] = sample.float().cpu().numpy()
            out[f"{name}_{b}x{n}_scale"] = np.float64(full.abs().double().mean().item())
    os.makedirs(out_dir, exist_ok=True)
    np.savez_compressed(os.path.join(out_dir, "network_ref.npz"), **out)
    print({k: np.shape(v) for k, v in out.items()})


if __name__ == "__main__":
    main(sys.argv[1])
