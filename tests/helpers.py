"""Shared helpers of the GPU parity tests (test infrastructure)."""
import importlib.util
import os

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_ref_ext = None
_ref_tried = False

# (n -> m, radii, nsamples) of the four SA levels (reference pvn3d.py:65-111)
SA_LEVELS = [(12288, 2048, (0.0175, 0.025), (16, 32)), (2048, 1024, (0.025, 0.05), (16, 32)),
             (1024, 512, (0.05, 0.1), (16, 32)), (512, 128, (0.1, 0.2), (16, 32))]


# the point columns of the Pointnet2MSG features stored in tests/golden/dropin_ref.npz (a fixed sample of 12288)
PN2MSG_POINTS = np.sort(np.random.default_rng(0).choice(12288, size=512, replace=False))[::2]


# DenseFusion + heads cases of tests/test_heads_gpu.py and tests/golden/heads_ref.npz
HEADS_CASES = [(2, 2048), (1, 12288), (2, 1000)]


def heads_modules():
    """DenseFusion + SEG / KpOF / CtrOf stacks in the reference's module layout, seeded, BN randomised (CPU)"""
    from pvn3d_b200 import heads, testing

    torch.manual_seed(3)
    mods = [m.eval() for m in heads.reference_layout_modules(22, 8)]
    for i, m in enumerate(mods):
        testing.randomize_bn_(m, 10 + i)
    return mods


def heads_inputs(b, n):
    """rgb_emb, cld_emb [b, 128, n] on the CPU (PointNet++ features are post-ReLU)"""
    g = torch.Generator().manual_seed(n)
    rgb_emb = torch.randn(b, 128, n, generator=g)
    return rgb_emb, torch.randn(b, 128, n, generator=g).abs()


def heads_points(n):
    """the point columns of the head outputs stored in tests/golden/heads_ref.npz"""
    return np.sort(np.random.default_rng(n).choice(n, size=min(n, 384), replace=False))


def sa_module_and_inputs():
    """the MSG set-abstraction module of the autograd drop-in test (this package's module, reference layout) and
    its inputs xyz [2, 512, 3], features [2, 6, 512], all on the CPU"""
    from pvn3d_b200.pointnet2 import PointnetSAModuleMSG

    torch.manual_seed(1)
    sa = PointnetSAModuleMSG(npoint=64, radii=[0.1, 0.2], nsamples=[8, 16], mlps=[[6, 16, 32], [6, 16, 32]]).eval()
    g = torch.Generator().manual_seed(3)
    return sa, torch.rand(2, 512, 3, generator=g), torch.rand(2, 6, 512, generator=g)


def sa_feature_grad(sa, xyz, feat):
    """d/dfeat of sum(out^2) through the module (fp32 cuDNN, TF32 off)"""
    feat = feat.clone().requires_grad_(True)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        _, out = sa(xyz, feat)
        out.square().sum().backward()
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    return feat.grad.detach()


def load_ref_ext():
    """The UNMODIFIED reference op library built by oracle/build_ref_ext.sh, or None."""
    global _ref_ext, _ref_tried
    if _ref_tried:
        return _ref_ext
    _ref_tried = True
    path = os.path.join(ROOT, "oracle", "_ref", "_ext.so")
    if not os.path.exists(path):
        return None
    try:
        spec = importlib.util.spec_from_file_location("_ext", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        _ref_ext = mod
    except Exception as e:  # pragma: no cover
        print("reference _ext not loadable:", e)
        _ref_ext = None
    return _ref_ext


def level_clouds(batch=2, seed0=500, shape="ycb", n=12288):
    """xyz of every SA level for `batch` synthetic frames, computed with the ORACLE's FPS."""
    from oracle import pn2
    from pvn3d_b200 import synth

    frames = [synth.make_frame(shape, n_points=n, seed=seed0 + i) for i in range(batch)]
    xyz = np.stack([f.pcld for f in frames])
    levels = [xyz]
    for (_, m, _, _) in SA_LEVELS:
        if levels[-1].shape[1] <= m:
            break
        idx = pn2.furthest_point_sampling(levels[-1], m)
        levels.append(np.take_along_axis(levels[-1], idx[..., None].astype(np.int64).repeat(3, -1), 1))
    return frames, levels


def t(x, dev):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


_ref_py = None
_ref_py_tried = False


def load_reference_python():
    """The UNMODIFIED reference Python staged by oracle/build_ref_ext.sh under oracle/_ref/py (lib/,
    common.py, datasets/ fixtures), imported on top of pvn3d_b200.compat.install() -- i.e. with this
    package's `_ext` bound at pointnet2_utils.py:19.  Returns a namespace of the reference modules, or
    None when the staging directory is absent."""
    global _ref_py, _ref_py_tried
    if _ref_py_tried:
        return _ref_py
    _ref_py_tried = True
    root = os.path.join(ROOT, "oracle", "_ref", "py")
    if not os.path.isdir(os.path.join(root, "lib")):
        return None
    import types

    from pvn3d_b200 import compat

    compat.install(root)
    try:
        from lib import pvn3d as ref_pvn3d
        from lib.pointnet2_utils import pointnet2_utils as ref_pn2_utils
        from lib.utils import basic_utils as ref_bu
        from lib.utils import meanshift_pytorch as ref_ms
        from lib.utils import pvn3d_eval_utils as ref_eval
    except Exception as e:  # pragma: no cover
        print("reference python not importable:", repr(e))
        return None
    _ref_py = types.SimpleNamespace(pvn3d=ref_pvn3d, pn2_utils=ref_pn2_utils, basic_utils=ref_bu,
                                    meanshift=ref_ms, eval_utils=ref_eval)
    return _ref_py
