"""DenseFusion + SEG / KpOF / CtrOf heads (SURVEY section 8 f3) on the tensor-core layer kernel against the
REFERENCE modules (pvn3d/lib/pvn3d.py:157-182,245-267,297-308): tests/golden/heads_ref.npz holds what the reference's
classes, with the weights of helpers.heads_modules, computed in fp32 (TF32 off) at a fixed sample of the points.

Tolerance: TF32 operands through 6 stacked 1x1 convolutions with K up to 1024 -> mean error <= 3e-3 and max error <=
3e-2 of the mean output magnitude per head (the class of the reference's default cuDNN TF32 path).
"""
import os

import numpy as np
import pytest
import torch

from pvn3d_b200 import eval_utils, fixtures, heads
from pvn3d_b200.eval_utils import FramePoseSolver

from helpers import HEADS_CASES, heads_inputs, heads_modules, heads_points

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref_modules(cuda_dev):
    return [m.to(cuda_dev).eval() for m in heads_modules()]


@pytest.fixture(scope="module")
def heads_golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "heads_ref.npz")))


@pytest.mark.parametrize("b,n", HEADS_CASES)
def test_fused_heads_match_reference_modules(cuda_dev, ref_modules, heads_golden, b, n):
    rgb_emb, cld_emb = (t.to(cuda_dev) for t in heads_inputs(b, n))
    eng = heads.FusedHeads(*ref_modules, device=cuda_dev)
    got = eng(rgb_emb, cld_emb)
    pts = torch.from_numpy(heads_points(n)).to(cuda_dev)
    samples = (got[0][:, :, pts], got[1][:, pts], got[2][:, :, pts])
    want = {}
    for name, full, gt in zip(("kp_of", "seg", "ctr_of"), got, samples):
        assert full.is_contiguous(), name
        w = torch.from_numpy(heads_golden[f"{name}_{b}x{n}"]).to(cuda_dev)
        want[name] = w
        assert gt.shape == w.shape, name
        scale = float(heads_golden[f"{name}_{b}x{n}_scale"])
        err = (gt - w).abs()
        print(f"{name} [{b}x{n}]: fused mean {float(err.mean()) / scale:.2e} max {float(err.max()) / scale:.2e}")
        assert float(err.mean()) <= 3e-3 * scale and float(err.max()) <= 3e-2 * scale, name
    assert got[0].shape == (b, 8, n, 3) and got[1].shape == (b, n, 22) and got[2].shape == (b, 1, n, 3)
    # the predicted classes agree wherever the reference's own margin is not a rounding artefact
    top2 = want["seg"].topk(2, dim=-1).values
    clear = (top2[..., 0] - top2[..., 1]) > 1e-2 * float(heads_golden[f"seg_{b}x{n}_scale"])
    assert torch.equal(samples[1].argmax(-1)[clear], want["seg"].argmax(-1)[clear])


def test_head_outputs_feed_the_pose_solver(cuda_dev, ref_modules):
    """network output -> seg argmax -> cal_frame_poses on device (demo.py:98-119 without the CNN): shapes and dtypes fit"""
    b, n = 1, 2048
    g = torch.Generator().manual_seed(1)
    eng = heads.FusedHeads(*ref_modules, device=cuda_dev)
    kp_of, seg, ctr_of = eng(torch.randn(b, 128, n, generator=g).to(cuda_dev), torch.randn(b, 128, n, generator=g).abs().to(cuda_dev))
    mask = eval_utils.seg_argmax(seg)
    assert mask.shape == (b, n) and mask.dtype == torch.int32
    pcld = torch.rand(b, n, 3, generator=g).to(cuda_dev)
    s = FramePoseSolver(b, n, 8, 22, fixtures.mesh_kps_table_ycb(), fixtures.radius_thresholds_ycb(), True, device=cuda_dev)
    poses, present, _, _ = s.solve(pcld, mask, ctr_of[:, 0].contiguous(), kp_of)
    torch.cuda.synchronize()
    assert poses.shape == (b, 22, 3, 4) and bool(torch.isfinite(poses).all())
