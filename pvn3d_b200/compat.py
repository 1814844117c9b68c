"""Drop this package into an unmodified checkout of the reference (ethnhe/PVN3D).

    import pvn3d_b200.compat as compat
    compat.install("/path/to/PVN3D/pvn3d")      # before `import lib...` / `python -m demo`

What install() does (SURVEY section 8b, App. D):
  1. registers pvn3d_b200._ext as `lib.pointnet2_utils._ext`, so the reference's
     pointnet2_utils.py:19 (`from lib.pointnet2_utils import _ext`) binds the sm_90a kernels;
  2. adds the small import shims the 2019 code needs on torch 2.x / PyYAML 6 (`torch._six`,
     `yaml.load` default Loader, empty `neupeak.utils.webcv2`, `plyfile`, `pcl` modules);
  3. with patch_post=True, after the reference modules are imported, rebinds
     `lib.utils.meanshift_pytorch.MeanShiftTorch` and
     `lib.utils.pvn3d_eval_utils.{MeanShiftTorch,cal_frame_poses,cal_frame_poses_lm}` to this
     package's implementations (demo.py:22 imports them by name -> call patch_post_modules()
     after importing demo, or import pvn3d_eval_utils first);
  4. with patch_model=True, rebinds `lib.pvn3d.PVN3D.forward` (patch_pvn3d_forward): in eval mode, without
     autograd and on CUDA inputs the network runs on FusedPVN3D (pvn3d_b200.network); anything else -- training,
     train_*.py, grad-enabled or CPU calls -- runs the reference's own forward.
Nothing here copies or edits reference files.
"""
from __future__ import annotations

import importlib
import itertools
import sys
import types


def _stub(name: str, **attrs) -> types.ModuleType:
    """Register a placeholder module `name` ONLY IF the real one cannot be imported: an installed (or
    already imported) package is never touched -- the reference loads meshes through plyfile.PlyData.read
    (basic_utils.py:109,468) and must keep the real reader when it is there."""
    mod = sys.modules.get(name)
    if mod is not None and not getattr(mod, "_pvn3d_b200_stub", False):
        return mod                       # real module (or somebody else's): leave it alone
    if mod is None:
        try:
            return importlib.import_module(name)
        except Exception:                # ImportError, or a package that fails to initialise here
            mod = types.ModuleType(name)
            mod._pvn3d_b200_stub = True
            sys.modules[name] = mod
    for k, v in attrs.items():
        if not hasattr(mod, k):
            setattr(mod, k, v)
    return mod


def install_import_shims() -> None:
    import torch

    if "torch._six" not in sys.modules:  # persistent_dataloader.py:17
        _stub("torch._six", string_classes=(str, bytes), int_classes=int, container_abcs=__import__("collections").abc)
    try:
        import yaml

        if not getattr(yaml.load, "_pvn3d_b200", False):
            _orig = yaml.load

            def _load(stream, Loader=None, **kw):  # common.py:133 calls yaml.load(f) without a Loader
                return _orig(stream, Loader=Loader or yaml.FullLoader, **kw)

            _load._pvn3d_b200 = True
            yaml.load = _load
    except ImportError:  # pragma: no cover
        pass
    noop = lambda *a, **k: None  # noqa: E731
    for pkg in ("neupeak", "neupeak.utils"):
        m = _stub(pkg)
        if getattr(m, "_pvn3d_b200_stub", False):
            m.__path__ = []
    _stub("neupeak.utils.webcv2", imshow=noop, waitKey=noop)  # meanshift_pytorch.py:9
    _stub("plyfile", PlyData=type("PlyData", (), {"read": staticmethod(noop)}))
    _stub("pcl")


def install(reference_root: str | None = None, patch_post: bool = False, patch_model: bool = False) -> None:
    from . import _ext

    install_import_shims()
    sys.modules["lib.pointnet2_utils._ext"] = _ext
    if reference_root is not None and reference_root not in sys.path:
        sys.path.insert(0, reference_root)
    if patch_post:
        patch_post_modules(import_missing=True)
    if patch_model:
        patch_pvn3d_forward(importlib.import_module("lib.pvn3d").PVN3D)


def _weights(model):
    """every parameter and buffer of the module tree, a DataParallel replica's included (replicate() keeps them as plain
    attributes, listed in _former_parameters, not in _parameters)"""
    for m in model.modules():
        for t in itertools.chain(m._parameters.values(), getattr(m, "_former_parameters", {}).values(), m._buffers.values()):
            if t is not None:
                yield t


def fused_engine(model, device):
    """The FusedPVN3D of `model` on `device`, cached in the module.  The cache key is (data_ptr, _version) of every
    parameter and buffer: load_state_dict, an optimiser step or a BatchNorm running-statistics update rebuilds the
    engine.  A DataParallel replica on the model's own device shares its tensors (and this cache) and hits it; replicas
    on other devices hold fresh copies and rebuild on every call -- run one process per GPU instead (pvn3d_b200.dist)."""
    from .network import FusedPVN3D

    key = tuple((t.data_ptr(), t._version) for t in _weights(model))
    cache = model.__dict__.setdefault("_pvn3d_b200_engines", {})   # plain attribute: copied by reference into replicas
    hit = cache.get(device)
    if hit is None or hit[0] != key:
        hit = cache[device] = (key, FusedPVN3D(model, device))
    return hit[1]


def patch_pvn3d_forward(cls) -> None:
    """Rebind cls.forward(pointcloud, rgb, choose) (the reference's PVN3D, or a class with the same forward) so that
    eval-mode, no-grad calls on CUDA inputs run fused_engine(self, device); every other call runs the original forward.
    Idempotent."""
    import torch

    if getattr(cls.forward, "_pvn3d_b200_orig", None) is not None:
        return
    orig = cls.forward

    def forward(self, pointcloud, rgb, choose):
        if self.training or torch.is_grad_enabled() or not (pointcloud.is_cuda and rgb.is_cuda and choose.is_cuda):
            return orig(self, pointcloud, rgb, choose)
        return fused_engine(self, pointcloud.device)(pointcloud, rgb, choose)

    forward._pvn3d_b200_orig = orig
    forward.__doc__ = orig.__doc__
    cls.forward = forward


def patch_post_modules(import_missing: bool = False) -> None:
    """Rebind the reference's post-processing entry points to the implementations of this package."""
    from . import eval_utils, meanshift

    targets = {
        "lib.utils.meanshift_pytorch": {"MeanShiftTorch": meanshift.MeanShiftTorch},
        "lib.utils.pvn3d_eval_utils": {
            "MeanShiftTorch": meanshift.MeanShiftTorch,
            "cal_frame_poses": eval_utils.cal_frame_poses,
            "cal_frame_poses_lm": eval_utils.cal_frame_poses_lm,
        },
        "demo": {
            "cal_frame_poses": eval_utils.cal_frame_poses,
            "cal_frame_poses_lm": eval_utils.cal_frame_poses_lm,
        },
    }
    for name, attrs in targets.items():
        mod = sys.modules.get(name)
        if mod is None and import_missing and name != "demo":
            try:
                mod = importlib.import_module(name)
            except Exception:  # reference not importable here: nothing to patch
                mod = None
        if mod is None:
            continue
        for k, v in attrs.items():
            setattr(mod, k, v)
