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
     autograd and on CUDA inputs the network runs on FusedPVN3D (pvn3d_b200.network), with bf16 heads inside a
     torch.autocast("cuda", dtype=torch.bfloat16) region and TF32 ones otherwise; anything else -- training,
     train_*.py, grad-enabled or CPU calls -- runs the reference's own forward;
  5. with patch_eval=True, rebinds `TorchEval.eval_pose_parallel` (patch_eval_pose_parallel): the poses of the whole
     batch in one FramePoseSolver.solve, every ground-truth object scored in one pvn3d_frame_add_adds launch, one
     device -> host read, and the distance lists appended exactly as eval_metric / eval_metric_lm would -- the
     reference's cal_auc / cal_lm_add then run unchanged;
  6. with patch_loss=True, rebinds `lib.loss.FocalLoss` / `lib.loss.OFLoss`, and the same names in
     `train.train_ycb_pvn3d` / `train.train_linemod_pvn3d` when those are already imported, to the drop-ins of
     pvn3d_b200.train_utils (import the training script first, then install).  get_item is not patched: it runs in
     forked DataLoader workers, where CUDA cannot start -- call train_utils.train_batch on the collated batch instead;
  7. with patch_vis=True, rebinds `lib.utils.basic_utils.Basic_Utils.draw_p2ds` on the class (patch_draw_p2ds), so the
     instance demo.py already holds draws on the GPU through pvn3d_b200.vis_utils.draw_p2ds; calls it cannot take run
     the reference's own method.
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


def install(reference_root: str | None = None, patch_post: bool = False, patch_model: bool = False,
            patch_eval: bool = False, patch_loss: bool = False, patch_vis: bool = False) -> None:
    from . import _ext

    install_import_shims()
    sys.modules["lib.pointnet2_utils._ext"] = _ext
    if reference_root is not None and reference_root not in sys.path:
        sys.path.insert(0, reference_root)
    if patch_post:
        patch_post_modules(import_missing=True)
    if patch_model:
        patch_pvn3d_forward(importlib.import_module("lib.pvn3d").PVN3D)
    if patch_eval:
        ev = importlib.import_module("lib.utils.pvn3d_eval_utils")
        patch_eval_pose_parallel(ev.TorchEval)
        for name in ("train.train_ycb_pvn3d", "train.train_linemod_pvn3d"):
            mod = sys.modules.get(name)
            if mod is not None and getattr(mod, "TorchEval", None) is not None:
                patch_eval_pose_parallel(mod.TorchEval)
    if patch_loss:
        patch_loss_modules()
    if patch_vis:
        patch_vis_modules()


def patch_vis_modules() -> None:
    """Rebind lib.utils.basic_utils.Basic_Utils.draw_p2ds (patch_draw_p2ds)."""
    patch_draw_p2ds(importlib.import_module("lib.utils.basic_utils").Basic_Utils)


def patch_draw_p2ds(cls) -> None:
    """Rebind cls.draw_p2ds(img, p2ds, r=1, color=(255, 0, 0)) (the reference's Basic_Utils, or a class with the same
    method) so that the calls vis_utils.gpu_drawable accepts -- a C-contiguous uint8 [H,W,3] image, int32 / int64
    [n,2] points, an integer r >= 0, a colour of 1 to 4 numbers, a CUDA device -- run vis_utils.draw_p2ds; every other
    call runs the original method.  Patched on the class, so existing instances pick it up.  Idempotent."""
    if getattr(cls.draw_p2ds, "_pvn3d_b200_orig", None) is not None:
        return
    orig = cls.draw_p2ds

    def draw_p2ds(self, img, p2ds, r=1, color=(255, 0, 0)):
        from . import vis_utils

        if not vis_utils.gpu_drawable(img, p2ds, r, color):
            return orig(self, img, p2ds, r, color)
        return vis_utils.draw_p2ds(img, p2ds, r, color)

    draw_p2ds._pvn3d_b200_orig = orig
    draw_p2ds.__doc__ = orig.__doc__
    cls.draw_p2ds = draw_p2ds


def patch_loss_modules() -> None:
    """Rebind FocalLoss and OFLoss in lib.loss and in the already imported training scripts to
    pvn3d_b200.train_utils's drop-ins (same constructors and forward signatures, CUDA only)."""
    from . import train_utils

    mods = [importlib.import_module("lib.loss")]
    mods += [sys.modules[m] for m in ("train.train_ycb_pvn3d", "train.train_linemod_pvn3d") if m in sys.modules]
    for mod in mods:
        for name in ("FocalLoss", "OFLoss"):
            if name in vars(mod):
                setattr(mod, name, getattr(train_utils, name))


def _weights(model):
    """every parameter and buffer of the module tree, a DataParallel replica's included (replicate() keeps them as plain
    attributes, listed in _former_parameters, not in _parameters)"""
    for m in model.modules():
        for t in itertools.chain(m._parameters.values(), getattr(m, "_former_parameters", {}).values(), m._buffers.values()):
            if t is not None:
                yield t


def fused_engine(model, device, precision="tf32"):
    """The FusedPVN3D of `model` on `device` at `precision`, cached in the module, one engine per (device, precision).
    The weight key is (data_ptr, _version) of every
    parameter and buffer: load_state_dict, an optimiser step or a BatchNorm running-statistics update rebuilds the
    engine.  A DataParallel replica on the model's own device shares its tensors (and this cache) and hits it; replicas
    on other devices hold fresh copies and rebuild on every call -- run one process per GPU instead (pvn3d_b200.dist)."""
    from .network import FusedPVN3D

    key = tuple((t.data_ptr(), t._version) for t in _weights(model))
    cache = model.__dict__.setdefault("_pvn3d_b200_engines", {})   # plain attribute: copied by reference into replicas
    hit = cache.get((device, precision))
    if hit is None or hit[0] != key:
        hit = cache[(device, precision)] = (key, FusedPVN3D(model, device, precision))
    return hit[1]


def autocast_precision() -> str:
    """the FusedPVN3D precision of a call made here: "bf16" inside torch.autocast("cuda", dtype=torch.bfloat16), "tf32"
    otherwise (fp16 autocast included: the library has no fp16 heads)"""
    import torch

    if torch.is_autocast_enabled("cuda") and torch.get_autocast_dtype("cuda") == torch.bfloat16:
        return "bf16"
    return "tf32"


def patch_pvn3d_forward(cls) -> None:
    """Rebind cls.forward(pointcloud, rgb, choose) (the reference's PVN3D, or a class with the same forward) so that
    eval-mode, no-grad calls on CUDA inputs run fused_engine(self, device, autocast_precision()); every other call runs
    the original forward.  Idempotent."""
    import torch

    if getattr(cls.forward, "_pvn3d_b200_orig", None) is not None:
        return
    orig = cls.forward

    def forward(self, pointcloud, rgb, choose):
        if self.training or torch.is_grad_enabled() or not (pointcloud.is_cuda and rgb.is_cuda and choose.is_cuda):
            return orig(self, pointcloud, rgb, choose)
        return fused_engine(self, pointcloud.device, autocast_precision())(pointcloud, rgb, choose)

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


def _batch_evaluator(ref, ds_type: str, obj_id: int, device):
    """the PoseEvaluator of one dataset (and LineMOD object) on `device`, cached in the reference module.  Meshes come
    from the reference's own bs_utils.get_pointxyz_cuda, once per class: LineMOD's loader draws a random 2000-point
    subset and caches it, so this evaluator and the reference's eval_metric_lm score the same points."""
    from .eval_utils import PoseEvaluator

    cache = ref.__dict__.setdefault("_pvn3d_b200_evaluators", {})
    key = (ds_type, obj_id if ds_type != "ycb" else None, str(device))
    ev = cache.get(key)
    if ev is None:
        if ds_type == "ycb":
            meshes = {c: ref.bs_utils.get_pointxyz_cuda(ref.cls_lst[c - 1]) for c in range(1, len(ref.cls_lst) + 1)}
            ev = PoseEvaluator(meshes, ref.config.ycb_sym_cls_ids, absent="zeros", device=device)
        else:
            mesh = ref.bs_utils_lm.get_pointxyz_cuda(obj_id, ds_type="linemod")
            ev = PoseEvaluator({1: mesh}, [], absent="identity", device=device)
        cache[key] = ev
    return ev


def patch_eval_pose_parallel(cls) -> None:
    """Rebind cls.eval_pose_parallel (the reference's TorchEval, pvn3d_eval_utils.py:345-387) to a batched form with
    the same arguments and the same effect on self.cls_add_dis / self.cls_adds_dis: cal_frame_poses(_lm) for every
    frame in one FramePoseSolver.solve (ds_type, use_ctr_clus_flter and obj_id as there), eval_metric(_lm) for every
    ground-truth object in one pvn3d_frame_add_adds launch, one device -> host read.  Idempotent."""
    if getattr(cls.eval_pose_parallel, "_pvn3d_b200_orig", None) is not None:
        return
    orig = cls.eval_pose_parallel
    ref = sys.modules[cls.__module__]

    def eval_pose_parallel(self, pclds, rgbs, masks, pred_ctr_ofs, gt_ctr_ofs, labels, cnt, cls_ids, RTs, pred_kp_ofs,
                           min_cnt=20, merge_clus=False, bbox=False, ds="YCB", cls_type=None, use_p2d=False,
                           vote_type=None, use_ctr_clus_flter=True, use_ctr=True, ds_type="ycb", obj_id=0):
        import torch

        from . import eval_utils

        if not use_ctr:
            raise NotImplementedError("use_ctr=False is never exercised by the reference callers")
        bs, n_kps, n_pts, _ = pred_kp_ofs.size()
        dev = pred_kp_ofs.device
        pcld = pclds.reshape(bs, n_pts, 3).float().contiguous()
        ctr = pred_ctr_ofs.reshape(bs, -1, n_pts, 3)[:, 0].float().contiguous()
        kp = pred_kp_ofs.float().contiguous()
        ycb = ds_type == "ycb"
        masks = masks.reshape(bs, n_pts)
        if ycb:
            m32 = masks.to(torch.int32).contiguous()
            s = eval_utils._solver("ycb", n_pts, n_kps, self.n_cls, bool(use_ctr_clus_flter), dev, batch=bs)
            gt, ids = RTs, cls_ids.reshape(bs, -1)
        else:
            m32 = (masks == 1).to(torch.int32).contiguous()      # cls_msk = mask == 1 (:171)
            s = eval_utils._solver("lm", n_pts, n_kps, max(self.n_cls, 2), bool(use_ctr_clus_flter), dev,
                                   obj_id=obj_id, batch=bs)     # the solver cal_frame_poses_lm uses, batched
            gt, ids = RTs[:, :1], torch.ones((bs, 1), dtype=torch.int32, device=dev)   # RTs[0] only (:211)
        ev = _batch_evaluator(ref, ds_type if ycb else "linemod", obj_id, dev)
        with s.lock:
            poses, present, _, _ = s.solve(pcld, m32, ctr, kp)
            if not ycb:
                poses, present = poses[:, :2], present[:, :2]          # class 1 only
            ev.reset()
            ev.add_batch(poses, present, gt, ids)
            add, adds = ev.distances()
        if ycb:
            for c in range(len(self.cls_add_dis)):
                self.cls_add_dis[c] += add[c] if c < len(add) else []
                self.cls_adds_dis[c] += adds[c] if c < len(adds) else []
        else:
            for dst, src in ((self.cls_add_dis, add), (self.cls_adds_dis, adds)):
                dst[obj_id] += src[1]
                dst[0] += src[0]

    eval_pose_parallel._pvn3d_b200_orig = orig
    eval_pose_parallel.__doc__ = orig.__doc__
    cls.eval_pose_parallel = eval_pose_parallel
