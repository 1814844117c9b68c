"""The UNMODIFIED reference Python running on this package's drop-in boundary, on the GPU.

oracle/build_ref_ext.sh stages the reference's lib/ + common.py + datasets/ fixtures under the
git-ignored oracle/_ref/py (it travels to the GPU box with the snapshot).  Here

  * the reference `Pointnet2MSG` (pvn3d/lib/pvn3d.py:46-154) -- its own pointnet2_utils.py /
    pointnet2_modules.py / pytorch_utils.py, nothing of this package's mirror -- runs with
    `lib.pointnet2_utils._ext` bound to pvn3d_b200._ext (pointnet2_utils.py:19) and must produce
    the SAME BITS as the same module object on the reference's own compiled `_ext`
    (oracle/_ref/_ext.so) with TF32 off: every index op is bit-exact, so every cuDNN call sees
    identical operands;
  * the reference `cal_frame_poses` / `cal_frame_poses_lm` (pvn3d_eval_utils.py:37-110,156-201),
    executed as written on CUDA tensors with the reference `MeanShiftTorch`, is compared with the
    same call after compat.patch_post_modules() (what demo.py:22,98-119 would run): class ids equal,
    poses within 1e-4.

Where the reference is not staged, this package's modules / entry points are compared with what the reference
computed on the same inputs (tests/golden/dropin_ref.npz).
"""
import os

import numpy as np
import pytest
import torch

from pvn3d_b200 import _ext as our_ext
from pvn3d_b200 import compat, synth, testing

from helpers import PN2MSG_POINTS, load_ref_ext, load_reference_python, sa_feature_grad, sa_module_and_inputs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref():
    """the staged reference modules, or None (the tests that can then use tests/golden/dropin_ref.npz)"""
    return load_reference_python()


@pytest.fixture(scope="module")
def ref_golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "dropin_ref.npz")))


def _mirror_features(dev, x):
    mine = testing.seeded_pointnet2msg(0, 1).to(dev)
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            return mine(x)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _pose_close(p, q, tol=1e-4):
    dr = np.linalg.norm(p[:, :3] - q[:, :3])
    dt = np.linalg.norm(p[:, 3] - q[:, 3]) / max(np.linalg.norm(q[:, 3]), 1e-9)
    return dr <= tol * np.sqrt(3) and dt <= tol, (dr, dt)


def test_reference_pointnet2msg_on_dropin_ext_is_bit_identical(cuda_dev, ref, ref_golden):
    frames = synth.make_batch("ycb", 2, n_points=12288, config_id=11)
    x = torch.from_numpy(np.stack([f.cld_rgb_nrm for f in frames])).to(cuda_dev)
    ref_ext = load_ref_ext()
    if ref is None or ref_ext is None:
        # the mirror on this package's ops against the stored reference features (reference module, reference _ext)
        y_ref = ref_golden["pn2msg_y"]
        y_mirror = _mirror_features(cuda_dev, x)[..., torch.from_numpy(PN2MSG_POINTS).to(cuda_dev)].cpu().numpy()
        assert y_mirror.shape == y_ref.shape == (2, 128, PN2MSG_POINTS.size)
        assert float(np.abs(y_mirror - y_ref).max()) <= 1e-3 * float(np.abs(y_ref).mean())
        return
    assert ref.pn2_utils._ext is our_ext, "compat.install() must have bound the drop-in at pointnet2_utils.py:19"
    torch.manual_seed(0)
    model = ref.pvn3d.Pointnet2MSG(input_channels=6)
    testing.randomize_bn_(model, 1)
    model = model.to(cuda_dev).eval()
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            y_ours = model(x)
            ref.pn2_utils._ext = ref_ext                     # the reference's own compiled kernels
            try:
                y_ref = model(x)
            finally:
                ref.pn2_utils._ext = our_ext
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    assert y_ours.shape == (2, 128, 12288)
    assert torch.equal(y_ours, y_ref), float((y_ours - y_ref).abs().max())
    # and the mirror module of this package (same state_dict) gives the same features
    y_mirror = _mirror_features(cuda_dev, x)
    assert float((y_mirror - y_ref).abs().max()) <= 1e-3 * float(y_ref.abs().mean())


def test_reference_sa_module_autograd_on_dropin_ext(cuda_dev, ref, ref_golden):
    """train_*.py path: autograd Functions call gather_points_grad / group_points_grad of the drop-in.  The feature
    gradient of an MSG set-abstraction module (weights of helpers.sa_module_and_inputs) through this package's module
    and autograd Functions on the drop-in must match the reference module on the reference's own compiled _ext
    (tests/golden/dropin_ref.npz); where the reference is staged, the reference's own autograd Functions on the
    drop-in are compared with it as well."""
    mine, xyz, feat = sa_module_and_inputs()
    xyz, feat = xyz.to(cuda_dev), feat.to(cuda_dev)
    want = torch.from_numpy(ref_golden["sa_grad"]).to(cuda_dev)
    grads = [sa_feature_grad(mine.to(cuda_dev).eval(), xyz, feat)]
    ref_ext = load_ref_ext()
    if ref is not None and ref_ext is not None:
        from lib.pointnet2_utils import pointnet2_modules as ref_mod

        sa = ref_mod.PointnetSAModuleMSG(npoint=64, radii=[0.1, 0.2], nsamples=[8, 16], mlps=[[6, 16, 32], [6, 16, 32]])
        sa.load_state_dict(mine.state_dict(), strict=True)
        sa = sa.to(cuda_dev).eval()
        for ext in (our_ext, ref_ext):
            ref.pn2_utils._ext = ext
            try:
                grads.append(sa_feature_grad(sa, xyz, feat))
            finally:
                ref.pn2_utils._ext = our_ext
    # scatter-adds accumulate in a different order: float tolerance, not bits
    for g in grads:
        assert torch.allclose(g, want, rtol=1e-4, atol=1e-5 * float(want.abs().max()))


@pytest.mark.parametrize("shape", ["ycb", "linemod"])
def test_reference_cal_frame_poses_vs_patched(cuda_dev, ref, ref_golden, shape):
    """reference post-processing on CUDA tensors (what demo.py runs) vs the same entry points after
    compat.patch_post_modules()"""
    f = synth.make_frame(shape, n_points=4096, seed=77, lm_obj_id=1 if shape == "linemod" else None)
    pcld = torch.from_numpy(f.pcld).to(cuda_dev)
    mask = torch.from_numpy(f.labels).to(cuda_dev)
    ctr_of = torch.from_numpy(f.ctr_of).to(cuda_dev)
    kp_of = torch.from_numpy(f.kp_of).to(cuda_dev)
    if ref is None:
        # this package's entry points (what patch_post_modules() installs) against the stored reference poses
        from pvn3d_b200 import eval_utils
        poses_ref = ref_golden[f"poses_{shape}"]
        if shape == "ycb":
            ids, poses = eval_utils.cal_frame_poses(pcld, mask, ctr_of, kp_of, True, 22, True)
            assert np.array_equal(np.asarray(ids, np.int64), ref_golden["ids_ycb"])
        else:
            poses = eval_utils.cal_frame_poses_lm(pcld, mask, ctr_of, kp_of, True, 2, False, 1)
        assert len(poses) == len(poses_ref)
        for p, q in zip(poses, poses_ref):
            ok, err = _pose_close(np.asarray(p, np.float64), q)
            assert ok, err
        return
    ev = ref.eval_utils
    orig = (ev.cal_frame_poses, ev.cal_frame_poses_lm, ev.MeanShiftTorch, ref.meanshift.MeanShiftTorch)
    if shape == "ycb":
        ids_ref, poses_ref = ev.cal_frame_poses(pcld, mask, ctr_of, kp_of, True, 22, True)
    else:
        poses_ref = ev.cal_frame_poses_lm(pcld, mask, ctr_of, kp_of, True, 2, False, 1)
    compat.patch_post_modules()
    try:
        assert ev.cal_frame_poses is not orig[0]
        if shape == "ycb":
            ids, poses = ev.cal_frame_poses(pcld, mask, ctr_of, kp_of, True, 22, True)
            assert np.array_equal(ids, ids_ref)
        else:
            poses = ev.cal_frame_poses_lm(pcld, mask, ctr_of, kp_of, True, 2, False, 1)
    finally:
        ev.cal_frame_poses, ev.cal_frame_poses_lm, ev.MeanShiftTorch, ref.meanshift.MeanShiftTorch = orig
    assert len(poses) == len(poses_ref)
    for p, q in zip(poses, poses_ref):
        # the reference ran torch CUDA kernels (soft cross-check: their norm / sum may round differently from
        # the CPU kernels the contract is pinned to), still well inside the bar
        ok, err = _pose_close(np.asarray(p, np.float64), np.asarray(q, np.float64))
        assert ok, err
