"""PVN3D's training targets and losses on the GPU (csrc/train.cu):

    targets = TrainTargets()                                   # YCB tables; TrainTargets.linemod(obj_id) for LineMOD
    batch = train_batch(builder, targets, depth, K, cam_scale, rgb, label_image, cls_ids, RTs, seed)
    rgb, pcld, cld_rgb_nrm, choose, kp_targ_ofst, ctr_targ_ofst, cls_ids, RTs, labels, kp3ds, ctr3ds, ok = batch
    loss, parts, acc = PVN3DLoss()(pred_kp_of, pred_rgbd_seg, pred_ctr_of, kp_targ_ofst, ctr_targ_ofst, labels, ok)

  * TrainTargets.compute is the target block of get_item (ycb_dataset.py:241-278, linemod_dataset.py:275-310) on the
    sampled cloud: pvn3d_train_targets, one launch.
  * train_batch fixes model_fn's 11-tuple (train_ycb_pvn3d.py:165-166) in one place: FrameInputBuilder.build with the
    label image, then the targets.  The DataLoader workers keep loading and decoding on the CPU (CUDA cannot start
    in forked workers); the main process augments the collated batch (augment.FrameAugmenter) and calls train_batch.
  * FocalLoss and OFLoss are drop-ins for lib/loss.py with its constructors and forward signatures, PVN3DLoss is
    model_fn's weighted sum of the three terms plus the accuracy; each is one torch.autograd.Function over
    pvn3d_train_loss_forward (two launches) and pvn3d_train_loss_backward (one launch), with no host sync.  They take
    CUDA tensors (float32; other float dtypes are upcast) and raise on CPU tensors: there is no CPU fallback.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch
from torch.nn.modules.loss import _Loss

from . import _lib, fixtures
from ._lib import LossArgs, check, ptr
from .icp import _aligned, _cuda_device

YCB_SLOTS = fixtures.YCB_N_CLASSES   #: config.n_objects: the meta slots of a YCB frame (common.py:51)
LM_SLOTS = 2                         #: LineMOD: n_objects = 2, slot 0 = the object, slot 1 empty (common.py:88)


def _cuda(t, what):
    if not torch.is_tensor(t) or not t.is_cuda:
        raise RuntimeError(f"{what} (pvn3d_b200): CUDA tensors only -- no CPU fallback")
    return t


def _f32(t, what):
    _cuda(t, what)
    if not t.is_floating_point():
        raise ValueError(f"{what}: expected a floating-point tensor, got {t.dtype}")
    return t.contiguous() if t.dtype == torch.float32 else t.float().contiguous()


def _int(t, dt, what):
    _cuda(t, what)
    if t.is_floating_point() or t.is_complex():
        raise ValueError(f"{what}: expected an integer tensor, got {t.dtype}")
    return t.to(dt).contiguous()


def _ids32(t, what):
    """integer class ids as int32 for the kernel; an id int32 cannot hold (an int64 label of 2**32 + 1, say) becomes
    -1, which matches no class and no slot -- as get_item's int64 comparison finds no match for it -- instead of
    wrapping onto a real class.  On the device, no host sync."""
    _cuda(t, what)
    if t.is_floating_point() or t.is_complex():
        raise ValueError(f"{what}: expected an integer tensor, got {t.dtype}")
    if t.dtype != torch.bool and (torch.iinfo(t.dtype).min < -2 ** 31 or torch.iinfo(t.dtype).max > 2 ** 31 - 1):
        t = torch.where((t >= -2 ** 31) & (t <= 2 ** 31 - 1), t, -1)
    return t.to(torch.int32).contiguous()


class TrainTargets:
    """get_item's regression targets on the GPU for a batch of sampled clouds.

    kp_table [n_cls,K,3] and ctr_table [n_cls,3] (float32) are the object-frame keypoints and centre of each class id,
    as Basic_Utils.get_kps / get_ctr load them; row 0 (background) is never read.  The defaults are the YCB tables of
    pvn3d_b200.fixtures (the K = 8 'farthest' set); any K works when a caller supplies its own tables."""

    def __init__(self, n_cls: int = None, kp_table=None, ctr_table=None, device="cuda"):
        self.dev = _cuda_device(device, "TrainTargets")
        if kp_table is None and ctr_table is None:
            t = fixtures.mesh_kps_table_ycb()
            kp_table, ctr_table = t[:, :fixtures.N_KEYPOINTS], t[:, fixtures.N_KEYPOINTS]
        kp = np.ascontiguousarray(kp_table, np.float32)
        ctr = np.ascontiguousarray(ctr_table, np.float32)
        if kp.ndim != 3 or kp.shape[2] != 3 or kp.shape[1] < 1 or ctr.shape != (kp.shape[0], 3):
            raise ValueError(f"TrainTargets: kp_table must be [n_cls,K,3] and ctr_table [n_cls,3], got {kp.shape} "
                             f"and {ctr.shape}")
        self.n_cls = kp.shape[0] if n_cls is None else int(n_cls)
        if self.n_cls != kp.shape[0] or self.n_cls < 2:
            raise ValueError(f"TrainTargets: n_cls={n_cls} but the tables have {kp.shape[0]} rows (at least 2)")
        self.k = kp.shape[1]
        self.kp_table = torch.from_numpy(kp).to(self.dev)
        self.ctr_table = torch.from_numpy(ctr).to(self.dev)
        self.lib = _lib.load()

    @classmethod
    def linemod(cls, obj_id: int, device="cuda") -> "TrainTargets":
        """the tables of LineMOD object `obj_id` at class id 1 (linemod_dataset.py's loop is enumerate([1]))"""
        t = fixtures.mesh_kps_table_lm(obj_id)
        return cls(2, t[:, :fixtures.N_KEYPOINTS], t[:, fixtures.N_KEYPOINTS], device)

    def compute(self, pcld, labels, cls_ids, RTs):
        """pcld [B,N,3] f32, labels [B,N] integer, cls_ids [B,S] or [B,S,1] integer (meta order, 0 = empty slot), RTs
        [B,S,3,4] (float64, as the meta poses get_item reads; float32 is widened) -> (kp_targ_ofst [B,N,K,3],
        ctr_targ_ofst [B,N,3], kp3ds [B,S,K,3], ctr3ds [B,S,3]), float32, on the current stream, no host sync."""
        pcld = _f32(pcld, "TrainTargets.compute: pcld")
        if pcld.dim() != 3 or pcld.size(2) != 3 or pcld.size(0) < 1 or pcld.size(1) < 1:
            raise ValueError(f"TrainTargets.compute: pcld must be [B,N,3], got {tuple(pcld.shape)}")
        b, n = pcld.shape[:2]
        if labels.shape != (b, n):
            raise ValueError(f"TrainTargets.compute: labels must be [{b},{n}], got {tuple(labels.shape)}")
        if cls_ids.dim() == 3 and cls_ids.size(2) == 1:
            cls_ids = cls_ids[..., 0]
        if cls_ids.dim() != 2 or cls_ids.size(0) != b or cls_ids.size(1) < 1:
            raise ValueError(f"TrainTargets.compute: cls_ids must be [{b},S] or [{b},S,1], got {tuple(cls_ids.shape)}")
        s = cls_ids.size(1)
        if RTs.shape != (b, s, 3, 4):
            raise ValueError(f"TrainTargets.compute: RTs must be [{b},{s},3,4], got {tuple(RTs.shape)}")
        for t, what in ((pcld, "pcld"), (labels, "labels"), (cls_ids, "cls_ids"), (RTs, "RTs")):
            _cuda(t, f"TrainTargets.compute: {what}")
            if t.device != self.dev:
                raise ValueError(f"TrainTargets.compute: {what} is on {t.device}, the tables on {self.dev}")
        lab = _ids32(labels, "TrainTargets.compute: labels")
        ids = _ids32(cls_ids, "TrainTargets.compute: cls_ids")
        if not RTs.is_floating_point():
            raise ValueError(f"TrainTargets.compute: RTs must be floating point, got {RTs.dtype}")
        rts = RTs.to(torch.float64).contiguous()
        f32 = dict(dtype=torch.float32, device=self.dev)
        kp_t = torch.empty((b, n, self.k, 3), **f32)
        ctr_t = torch.empty((b, n, 3), **f32)
        kp3 = torch.empty((b, s, self.k, 3), **f32)
        ctr3 = torch.empty((b, s, 3), **f32)
        with torch.cuda.device(self.dev):
            rc = self.lib.pvn3d_train_targets(ptr(pcld), ptr(lab), ptr(ids), ptr(rts), b, n, s, ptr(self.kp_table),
                                              ptr(self.ctr_table), self.n_cls, self.k, ptr(kp_t), ptr(ctr_t), ptr(kp3),
                                              ptr(ctr3), torch.cuda.current_stream(self.dev).cuda_stream)
        check(rc, "pvn3d_train_targets")
        return kp_t, ctr_t, kp3, ctr3


def train_batch(builder, targets: TrainTargets, depth, K, cam_scale, rgb, label_image, cls_ids, RTs, seed: int):
    """model_fn's batch (train_ycb_pvn3d.py:165-166) from raw frames, on the GPU: FrameInputBuilder.build(...,
    label_image=) then TrainTargets.compute on the builder's own pcld and labels.  cls_ids [B,S] (or [B,S,1]) and RTs
    [B,S,3,4] are the collated meta slots (float64 poses for get_item's float64 targets).

    Returns (rgb [B,3,H,W] f32, pcld [B,N,3] f32, cld_rgb_nrm [B,N,9] f32, choose [B,1,N] i64, kp_targ_ofst
    [B,N,K,3] f32, ctr_targ_ofst [B,N,3] f32, cls_ids [B,S,1] i64, RTs [B,S,3,4] f32, labels [B,N] i64, kp3ds [B,S,K,3]
    f32, ctr3ds [B,S,3] f32) -- get_item's outputs in its order and dtypes, batched -- and ok [B] u8.  A frame with
    ok = 0 (fewer than 400 valid pixels, which get_item would have dropped) has zero points, labels and offsets.
    Builder outputs are views of its buffers (valid until its next build); no host sync."""
    cld, rgb_o, choose, pcld, ok, labels = builder.build(depth, K, cam_scale, rgb, seed, label_image=label_image)
    if cls_ids.dim() == 2:
        cls_ids = cls_ids[..., None]
    kp_t, ctr_t, kp3, ctr3 = targets.compute(pcld, labels, cls_ids, RTs)
    return (rgb_o, pcld, cld, choose, kp_t, ctr_t, cls_ids.to(torch.int64), RTs.to(torch.float32),
            labels.to(torch.int64), kp3, ctr3, ok)


# ---------------------------------------------------------------------------------------------------------------------
# losses
# ---------------------------------------------------------------------------------------------------------------------

class _Spec:
    """the non-tensor arguments of one loss call"""

    def __init__(self, gamma=0.0, seg_mean=True, inner=1, weights=(1.0, 1.0, 1.0), b=0, n=0):
        self.gamma, self.seg_mean, self.inner, self.weights, self.b, self.n = float(gamma), bool(seg_mean), int(inner), \
            tuple(float(w) for w in weights), int(b), int(n)


def _args(spec, seg, seg_target, kp_pred, kp_targ, ctr_pred, ctr_targ, labels, ok) -> LossArgs:
    a = LossArgs()
    if seg is not None:
        a.seg, a.seg_target = ptr(seg), ptr(seg_target)
        a.seg_rows = seg_target.numel()
        a.n_cls = seg.size(1)
        a.seg_inner, a.gamma, a.seg_mean = spec.inner, spec.gamma, int(spec.seg_mean)
    if kp_pred is not None:
        a.kp_pred, a.kp_targ, a.n_kp = ptr(kp_pred), ptr(kp_targ), kp_pred.size(1)
    if ctr_pred is not None:
        a.ctr_pred, a.ctr_targ, a.n_ctr = ptr(ctr_pred), ptr(ctr_targ), ctr_pred.size(1)
    a.labels, a.b, a.n, a.ok = ptr(labels), spec.b, spec.n, ptr(ok)
    a.w_seg, a.w_kp, a.w_ctr = spec.weights
    return a


class _TrainLoss(torch.autograd.Function):
    """(loss [], parts [3], kp_loss [b,n_kp] (empty without a kp term), acc []) of the enabled terms"""

    @staticmethod
    def forward(ctx, spec, seg, kp_pred, ctr_pred, seg_target, kp_targ, ctr_targ, labels, ok):
        lib = _lib.load()
        t0 = next(t for t in (seg, kp_pred, ctr_pred) if t is not None)
        dev = t0.device
        a = _args(spec, seg, seg_target, kp_pred, kp_targ, ctr_pred, ctr_targ, labels, ok)
        nbytes = int(lib.pvn3d_train_loss_workspace_bytes(ctypes.byref(a)))
        if nbytes == 0:
            raise ValueError("pvn3d_train_loss: inconsistent arguments")
        ws, ws_ptr = _aligned(nbytes, dev)
        f32 = dict(dtype=torch.float32, device=dev)
        loss, parts, acc = torch.empty((), **f32), torch.empty((3,), **f32), torch.empty((), **f32)
        kp_loss = torch.empty((spec.b, kp_pred.size(1)) if kp_pred is not None else (0,), **f32)
        with torch.cuda.device(dev):
            rc = lib.pvn3d_train_loss_forward(ctypes.byref(a), ptr(loss), ptr(parts), ptr(kp_loss) if kp_pred is not None
                                              else 0, 0, ptr(acc), ws_ptr, nbytes,
                                              torch.cuda.current_stream(dev).cuda_stream)
        check(rc, "pvn3d_train_loss_forward")
        ctx.spec, ctx.ws, ctx.ws_ptr, ctx.nbytes = spec, ws, ws_ptr, nbytes
        ctx.save_for_backward(seg, kp_pred, ctr_pred, seg_target, kp_targ, ctr_targ, labels, ok)
        ctx.mark_non_differentiable(acc)
        ctx.set_materialize_grads(False)
        return loss, parts, kp_loss, acc

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_loss, g_parts, g_kp, _g_acc):
        seg, kp_pred, ctr_pred, seg_target, kp_targ, ctr_targ, labels, ok = ctx.saved_tensors
        if g_loss is None and g_parts is None and g_kp is None:
            return (None,) * 9
        g = [None if x is None else x.float().contiguous() for x in (g_loss, g_parts, g_kp)]
        d_seg = None if seg is None else torch.empty_like(seg)
        d_kp = None if kp_pred is None else torch.empty_like(kp_pred)
        d_ctr = None if ctr_pred is None else torch.empty_like(ctr_pred)
        a = _args(ctx.spec, seg, seg_target, kp_pred, kp_targ, ctr_pred, ctr_targ, labels, ok)
        dev = ctx.ws.device
        with torch.cuda.device(dev):
            rc = _lib.load().pvn3d_train_loss_backward(ctypes.byref(a), ptr(g[0]), ptr(g[1]), ptr(g[2]), ptr(d_seg),
                                                       ptr(d_kp), ptr(d_ctr), ctx.ws_ptr, ctx.nbytes,
                                                       torch.cuda.current_stream(dev).cuda_stream)
        check(rc, "pvn3d_train_loss_backward")
        return None, d_seg, d_kp, d_ctr, None, None, None, None, None


def _of_inputs(pred, targ, labels, what):
    pred = _f32(pred, f"{what}: pred_ofsts")
    if pred.dim() != 4 or pred.size(3) != 3:
        raise ValueError(f"{what}: pred_ofsts must be [bs,n_kpts,n_pts,3], got {tuple(pred.shape)}")
    bs, n_kpts, n_pts, _ = pred.shape
    targ = _f32(targ, f"{what}: targ_ofst")
    if targ.numel() != pred.numel():
        raise ValueError(f"{what}: targets must hold bs*n_pts*n_kpts*3 = {pred.numel()} values "
                         f"(.view(bs, n_pts, n_kpts, 3)), got {tuple(targ.shape)}")
    _cuda(labels, f"{what}: labels")
    if labels.numel() != bs * n_pts:
        raise ValueError(f"{what}: labels must hold bs*n_pts = {bs * n_pts} values, got {tuple(labels.shape)}")
    if labels.is_floating_point():
        labels = labels > 1e-8                      # w = (labels > 1e-8): the kernel takes labels > 0
    lab = _int(labels.reshape(bs, n_pts), torch.int64, f"{what}: labels")
    for t in (targ, lab):
        if t.device != pred.device:
            raise ValueError(f"{what}: every input must be on {pred.device}")
    return pred, targ.view(bs, n_pts, n_kpts, 3), lab


def _seg_inputs(logits, target, what):
    x = _f32(logits, f"{what}: input")
    if x.dim() < 2:
        raise ValueError(f"{what}: input must be [M,C] or [N,C,...], got {tuple(x.shape)}")
    inner = 1
    if x.dim() > 2:                                  # N,C,H,W => N*H*W rows, read in place (no transpose copy)
        inner = int(np.prod(x.shape[2:]))
    rows = x.size(0) * inner
    _cuda(target, f"{what}: target")
    if target.numel() != rows or rows < 1 or inner < 1:
        raise ValueError(f"{what}: target must hold {rows} class ids, got {tuple(target.shape)}")
    t = _int(target.reshape(-1), torch.int64, f"{what}: target")
    if t.device != x.device:
        raise ValueError(f"{what}: input and target must be on the same device")
    return x.reshape(x.size(0), x.size(1), inner) if inner > 1 else x, t, inner


class FocalLoss(_Loss):
    """lib/loss.py's FocalLoss on the GPU: the mean (size_average) or sum over rows of -(1-pt)^gamma log(pt), with pt
    detached as the reference's Variable(logpt.data.exp()) makes it.  input [M,C] or [N,C,*] (reshaped to N*H*W rows as
    the reference does), target integer class ids; a target outside [0, C) gives NaN (the reference's gather asserts)."""

    def __init__(self, gamma=0, alpha=None, size_average=True):
        super().__init__()
        if alpha is not None:
            raise ValueError("FocalLoss (pvn3d_b200): alpha is not supported (PVN3D never sets it)")
        if not float(gamma) >= 0 or not np.isfinite(float(gamma)):
            raise ValueError(f"FocalLoss (pvn3d_b200): gamma={gamma} must be finite and >= 0")
        self.gamma, self.alpha, self.size_average = gamma, alpha, size_average

    def forward(self, input, target):
        x, t, inner = _seg_inputs(input, target, "FocalLoss")
        spec = _Spec(gamma=self.gamma, seg_mean=self.size_average, inner=inner)
        return _TrainLoss.apply(spec, x, None, None, t, None, None, None, None)[0]


class OFLoss(_Loss):
    """lib/loss.py's OFLoss on the GPU: [bs, n_kpts] = sum_{n,c} w |pred - targ| / (sum_n w + 1e-3), w = labels > 1e-8.
    pred_ofsts [bs,n_kpts,n_pts,3], kp_targ_ofst viewed as [bs,n_pts,n_kpts,3], labels [bs,n_pts] (any shape with that
    many values).  normalize / reduce are accepted and ignored, as the reference's forward ignores them."""

    def __init__(self):
        super().__init__()

    def forward(self, pred_ofsts, kp_targ_ofst, labels, normalize=True, reduce=False):
        pred, targ, lab = _of_inputs(pred_ofsts, kp_targ_ofst, labels, "OFLoss")
        spec = _Spec(b=pred.size(0), n=pred.size(2))
        return _TrainLoss.apply(spec, None, pred, None, None, targ, None, lab, None)[2]


class PVN3DLoss(torch.nn.Module):
    """model_fn's loss (train_ycb_pvn3d.py:172-184) in one forward chain and one backward launch:
    loss = w0 FocalLoss(gamma)(seg, labels) + w1 sum(OFLoss(kp)) + w2 sum(OFLoss(ctr)).

    forward(pred_kp_of [B,K,N,3], pred_rgbd_seg [B,N,C], pred_ctr_of [B,1,N,3], kp_targ_ofst [B,N,K,3],
    ctr_targ_ofst [B,N,3], labels [B,N], ok=None) -> (loss [], parts [3] = (focal, sum kp, sum ctr), acc []), device
    tensors.  acc = share of rows whose first argmax equals the label.  ok [B] (FrameInputBuilder's) leaves the rows
    of ok = 0 frames out of the focal mean and the accuracy; with no ok frame, loss and gradient are 0."""

    def __init__(self, weights=(2.0, 1.0, 1.0), gamma=2):
        super().__init__()
        if len(weights) != 3:
            raise ValueError(f"PVN3DLoss: weights must be 3 numbers, got {weights}")
        if not float(gamma) >= 0 or not np.isfinite(float(gamma)):
            raise ValueError(f"PVN3DLoss: gamma={gamma} must be finite and >= 0")
        self.weights, self.gamma = tuple(float(w) for w in weights), float(gamma)

    def forward(self, pred_kp_of, pred_rgbd_seg, pred_ctr_of, kp_targ_ofst, ctr_targ_ofst, labels, ok=None):
        kp, kt, lab = _of_inputs(pred_kp_of, kp_targ_ofst, labels, "PVN3DLoss (kp)")
        ctr, ct, _ = _of_inputs(pred_ctr_of, ctr_targ_ofst, labels, "PVN3DLoss (ctr)")
        b, n = kp.size(0), kp.size(2)
        if ctr.shape[0] != b or ctr.shape[2] != n:
            raise ValueError(f"PVN3DLoss: pred_ctr_of {tuple(ctr.shape)} does not match pred_kp_of {tuple(kp.shape)}")
        seg = _f32(pred_rgbd_seg, "PVN3DLoss: pred_rgbd_seg")
        if seg.numel() % (b * n) != 0 or seg.numel() == 0:
            raise ValueError(f"PVN3DLoss: pred_rgbd_seg must be [{b},{n},C], got {tuple(seg.shape)}")
        seg = seg.reshape(b * n, -1)
        okb = None
        if ok is not None:
            _cuda(ok, "PVN3DLoss: ok")
            if ok.numel() != b:
                raise ValueError(f"PVN3DLoss: ok must hold {b} flags, got {tuple(ok.shape)}")
            okb = (ok.reshape(b) != 0).to(torch.uint8) if ok.dtype != torch.uint8 else ok.reshape(b).contiguous()
        for t in (seg, ctr, okb):
            if t is not None and t.device != kp.device:
                raise ValueError(f"PVN3DLoss: every input must be on {kp.device}")
        spec = _Spec(gamma=self.gamma, weights=self.weights, b=b, n=n)
        loss, parts, _, acc = _TrainLoss.apply(spec, seg, kp, ctr, lab.reshape(-1), kt, ct, lab, okb)
        return loss, parts, acc
