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
     after importing demo, or import pvn3d_eval_utils first).
Nothing here copies or edits reference files.
"""
from __future__ import annotations

import importlib
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


def install(reference_root: str | None = None, patch_post: bool = False) -> None:
    from . import _ext

    install_import_shims()
    sys.modules["lib.pointnet2_utils._ext"] = _ext
    if reference_root is not None and reference_root not in sys.path:
        sys.path.insert(0, reference_root)
    if patch_post:
        patch_post_modules(import_missing=True)


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
