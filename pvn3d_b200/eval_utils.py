"""cal_frame_poses / cal_frame_poses_lm / best_fit_transform -- drop-ins for the reference's
post-network pose recovery (pvn3d/lib/utils/pvn3d_eval_utils.py:37-110,156-201 and
pvn3d/lib/utils/basic_utils.py:47-80), executed by csrc/poses.cu + csrc/meanshift.cu.

Reference-compatible entry points (same arguments, same return types):
    cal_frame_poses(pcld, mask, ctr_of, pred_kp_of, use_ctr, n_cls, use_ctr_clus_flter)
        -> (pred_cls_ids: np.ndarray, pred_pose_lst: list[np.ndarray(3,4) float64])
    cal_frame_poses_lm(pcld, mask, ctr_of, pred_kp_of, use_ctr, n_cls, use_ctr_clus_flter, obj_id)
        -> list[np.ndarray(3,4) float64]
    best_fit_transform(A, B) -> np.ndarray(3,4) float64
Batched, sync-free form used by the frame pipeline and bench.py:
    FramePoseSolver(...).solve(pcld[B,N,3], mask[B,N], ctr_of[B,N,3], kp_of[B,K,N,3])
Scoring (TorchEval's eval_metric / eval_metric_lm / cal_auc / cal_lm_add, pvn3d_eval_utils.py:113-137,204-343):
    PoseEvaluator(meshes, sym_cls_ids, diameters, absent).add_batch(poses, present, gt_rt, cls_ids)
    -> .distances() / .auc() / .lm_accuracy(cls)
"""
from __future__ import annotations

import threading
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib, fixtures
from ._lib import check, ms_flags, ptr

RADIUS = 0.08  # clustering bandwidth hard-coded by the reference (pvn3d_eval_utils.py:44,163)


class FramePoseSolver:
    """Device-resident solver for a fixed (B, N, K, n_cls) problem shape; owns its workspace."""

    def __init__(self, batch: int, n_pts: int, n_kps: int, n_cls: int, mesh_kps: np.ndarray,
                 cls_radius: Optional[np.ndarray], use_ctr_clus_flter: bool, device="cuda",
                 bandwidth: float = RADIUS, max_iter: int = 300, early_exit: bool = False, mode: str = None):
        self.lib = _lib.load()
        self.dev = torch.device(device)
        if self.dev.type != "cuda":
            raise RuntimeError("FramePoseSolver: CUDA only -- no CPU fallback")
        self.b, self.n, self.k, self.n_cls = int(batch), int(n_pts), int(n_kps), int(n_cls)
        mesh_kps = np.ascontiguousarray(mesh_kps, dtype=np.float32)
        assert mesh_kps.shape == (self.n_cls, self.k + 1, 3), mesh_kps.shape
        self.mesh_kps = torch.from_numpy(mesh_kps).to(self.dev)
        self.use_filter = bool(use_ctr_clus_flter)
        self.cls_radius = None
        if self.use_filter:
            assert cls_radius is not None and len(cls_radius) == self.n_cls
            self.cls_radius = torch.from_numpy(np.ascontiguousarray(cls_radius, dtype=np.float32)).to(self.dev)
        self.bandwidth, self.max_iter = float(bandwidth), int(max_iter)
        self.flags = ms_flags(mode, early_exit)       # default: "certified" (see MeanShiftTorch)
        self.ws_bytes = int(self.lib.pvn3d_frame_poses_workspace_bytes(self.b, self.n, self.k, self.n_cls, self.max_iter))
        self._ws = torch.empty((self.ws_bytes + 256,), dtype=torch.uint8, device=self.dev)
        self._ws_ptr = (self._ws.data_ptr() + 255) // 256 * 256
        self.poses = torch.empty((self.b, self.n_cls, 3, 4), dtype=torch.float32, device=self.dev)
        self.present = torch.empty((self.b, self.n_cls), dtype=torch.uint8, device=self.dev)
        self.cls_kps = torch.empty((self.b, self.n_cls, self.k + 1, 3), dtype=torch.float32, device=self.dev)
        self.new_mask = torch.empty((self.b, self.n), dtype=torch.int32, device=self.dev)
        self._ms_off = int(self.lib.pvn3d_frame_poses_ms_workspace_offset(self.b, self.n, self.k, self.n_cls, self.max_iter))

    def certified_fits(self) -> int:
        """diagnostics (synchronises): how many of the last solve()'s centre + keypoint fits the witness
        kernel closed without sweeping all seeds (mode "certified")"""
        off = self._ws_ptr - self._ws.data_ptr() + self._ms_off
        return int(self._ws[off:off + 64].view(torch.int32)[_lib.PVN3D_MS_STAT_CERTIFIED].item())

    def solve(self, pcld: torch.Tensor, mask: torch.Tensor, ctr_of: torch.Tensor, kp_of: torch.Tensor):
        """All inputs on device, contiguous: pcld [B,N,3] f32, mask [B,N] i32, ctr_of [B,N,3] f32,
        kp_of [B,K,N,3] f32.  Returns (poses [B,n_cls,3,4], present [B,n_cls] u8, cls_kps, new_mask)
        -- views of solver-owned buffers, valid until the next solve() on the same stream."""
        b = pcld.size(0)
        assert b <= self.b and pcld.shape[1:] == (self.n, 3) and kp_of.shape[1:] == (self.k, self.n, 3)
        for t, dt in ((pcld, torch.float32), (mask, torch.int32), (ctr_of, torch.float32), (kp_of, torch.float32)):
            assert t.is_cuda and t.is_contiguous() and t.dtype == dt
        with torch.cuda.device(self.dev):
            rc = self.lib.pvn3d_frame_poses_batch(
                ptr(pcld), ptr(mask), ptr(ctr_of), ptr(kp_of), b, self.n, self.k, self.n_cls,
                ptr(self.mesh_kps), ptr(self.cls_radius), 1 if self.use_filter else 0,
                self.bandwidth, self.max_iter, self.flags, ptr(self.poses), ptr(self.present),
                ptr(self.cls_kps), ptr(self.new_mask), self._ws_ptr, self.ws_bytes,
                torch.cuda.current_stream(self.dev).cuda_stream)
        check(rc, "pvn3d_frame_poses_batch")
        return self.poses[:b], self.present[:b], self.cls_kps[:b], self.new_mask[:b]


_solver_cache = {}
_solver_cache_lock = threading.Lock()


def _solver(kind, n_pts, n_kps, n_cls, use_filter, dev, obj_id=None, early_exit=False, mode=None, batch=1):
    """the cached solver of one problem shape (batch 1 for the per-frame entry points).  Its output buffers are shared by every caller: hold
    `solver.lock` from solve() until the outputs have been copied out (the reference calls cal_frame_poses from a
    thread pool, pvn3d_eval_utils.py:373-380)."""
    key = (kind, batch, n_pts, n_kps, n_cls, use_filter, str(dev), obj_id, ms_flags(mode, early_exit))
    with _solver_cache_lock:
        s = _solver_cache.get(key)
        if s is None:
            if kind == "ycb":
                mesh = fixtures.mesh_kps_table_ycb()[:n_cls]
                rad = fixtures.radius_thresholds_ycb()[:n_cls] if use_filter else None
            else:
                mesh = np.zeros((n_cls, n_kps + 1, 3), np.float32)
                mesh[1] = fixtures.mesh_kps_table_lm(obj_id)[1]
                rad = np.full((n_cls,), np.inf, np.float32) if use_filter else None
            s = FramePoseSolver(batch, n_pts, n_kps, n_cls, mesh, rad, use_filter, device=dev, early_exit=early_exit,
                                mode=mode)
            s.lock = threading.Lock()
            _solver_cache[key] = s
    return s


def _prep(pcld, mask, ctr_of, pred_kp_of):
    if not pcld.is_cuda:
        raise RuntimeError("cal_frame_poses (pvn3d_b200): CUDA tensors only -- no CPU fallback")
    n_kps, n_pts, _ = pred_kp_of.size()
    return (pcld.reshape(1, n_pts, 3).contiguous().float(), ctr_of[0].reshape(1, n_pts, 3).contiguous().float(),
            pred_kp_of.reshape(1, n_kps, n_pts, 3).contiguous().float(), n_kps, n_pts)


def cal_frame_poses(pcld, mask, ctr_of, pred_kp_of, use_ctr, n_cls, use_ctr_clus_flter,
                    early_exit: bool = False, mode: str = None) -> Tuple[np.ndarray, List[np.ndarray]]:
    """pvn3d_eval_utils.py:37-110.  pcld [N,3], mask [N] (int64 class ids), ctr_of [1,N,3],
    pred_kp_of [K,N,3]; one device->host read at the end instead of >= 3 per class."""
    if not use_ctr:
        raise NotImplementedError("use_ctr=False is never exercised by the reference callers")
    p, c, kp, n_kps, n_pts = _prep(pcld, mask, ctr_of, pred_kp_of)
    m32 = mask.reshape(1, n_pts).to(torch.int32).contiguous()
    s = _solver("ycb", n_pts, n_kps, int(n_cls), bool(use_ctr_clus_flter), pcld.device, early_exit=early_exit,
                mode=mode)
    with s.lock:                       # the solver's buffers stay ours until the host copies are done
        poses, present, _, _ = s.solve(p, m32, c, kp)
        poses_h = poses[0].double().cpu().numpy()
        present_h = present[0].cpu().numpy()
    pred_cls_ids = np.nonzero(present_h)[0].astype(np.int64)  # == np.unique(mask[mask>0]) (:50)
    return pred_cls_ids, [poses_h[c_id].copy() for c_id in pred_cls_ids]


def cal_frame_poses_lm(pcld, mask, ctr_of, pred_kp_of, use_ctr, n_cls, use_ctr_clus_flter, obj_id,
                       early_exit: bool = False, mode: str = None) -> List[np.ndarray]:
    """pvn3d_eval_utils.py:156-201: single class id 1, fixtures of LineMOD object `obj_id`."""
    if not use_ctr:
        raise NotImplementedError("use_ctr=False is never exercised by the reference callers")
    p, c, kp, n_kps, n_pts = _prep(pcld, mask, ctr_of, pred_kp_of)
    m32 = (mask.reshape(1, n_pts) == 1).to(torch.int32).contiguous()  # cls_msk = mask == 1 (:169-170)
    # the lm variant has no centre-cluster relabel pass; the flag only gates the inlier filter of
    # the keypoint votes (:182-185), which the solver's flag also controls -> give it an infinite
    # radius so the relabel pass is the identity.
    s = _solver("lm", n_pts, n_kps, max(int(n_cls), 2), bool(use_ctr_clus_flter), pcld.device, obj_id=obj_id,
                early_exit=early_exit, mode=mode)
    with s.lock:
        poses, _, _, _ = s.solve(p, m32, c, kp)
        return [poses[0, 1].double().cpu().numpy()]


def best_fit_transform(A, B) -> np.ndarray:
    """basic_utils.py:47-80: least-squares rigid transform mapping A [P,3] onto B [P,3] -> 3x4 float64.
    Accepts numpy arrays or tensors; the SVD runs on the GPU (float64)."""
    lib = _lib.load()
    a = torch.as_tensor(np.asarray(A, dtype=np.float32) if not torch.is_tensor(A) else A.float())
    b = torch.as_tensor(np.asarray(B, dtype=np.float32) if not torch.is_tensor(B) else B.float())
    assert a.shape == b.shape and a.dim() == 2 and a.size(1) == 3
    a = a.cuda().contiguous()
    b = b.cuda().contiguous()
    rt = torch.empty((1, 3, 4), dtype=torch.float32, device=a.device)
    with torch.cuda.device(a.device):
        rc = lib.pvn3d_best_fit_transform_batch(ptr(a), ptr(b), 0, 1, int(a.size(0)), ptr(rt),
                                                torch.cuda.current_stream(a.device).cuda_stream)
    check(rc, "pvn3d_best_fit_transform_batch")
    return rt[0].double().cpu().numpy()


# --------------------------------------------------------------------------------------------------
# callers either side of the path (SURVEY section 8 f4): segmentation argmax, ADD / ADD-S
# --------------------------------------------------------------------------------------------------
def seg_argmax(logits: torch.Tensor) -> torch.Tensor:
    """`_, classes_rgbd = torch.max(pred_rgbd_seg, -1)` (demo.py:108) as one kernel: logits [..., n_cls] f32
    -> int32 class ids [...] -- the `mask` FramePoseSolver.solve takes (first maximal index)."""
    if not logits.is_cuda:
        raise RuntimeError("seg_argmax (pvn3d_b200): CUDA tensors only -- no CPU fallback")
    lib = _lib.load()
    x = logits.contiguous().float()
    n_cls = x.size(-1)
    out = torch.empty(x.shape[:-1], dtype=torch.int32, device=x.device)
    with torch.cuda.device(x.device):
        rc = lib.pvn3d_seg_argmax(ptr(x), x.numel() // n_cls, n_cls, ptr(out), torch.cuda.current_stream(x.device).cuda_stream)
    check(rc, "pvn3d_seg_argmax")
    return out


def pose_add_adds(pred_RT: torch.Tensor, gt_RT: torch.Tensor, p3ds: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """ADD and ADD-S of F pose pairs over one mesh in two launches: pred_RT, gt_RT [F,3,4] (or [3,4]),
    p3ds [P,3] -> (add [F], adds [F]).  basic_utils.py:617-635."""
    if not p3ds.is_cuda:
        raise RuntimeError("pose_add_adds (pvn3d_b200): CUDA tensors only -- no CPU fallback")
    lib = _lib.load()
    dev = p3ds.device
    pr = pred_RT.reshape(-1, 3, 4).to(dev, torch.float32).contiguous()
    gt = gt_RT.reshape(-1, 3, 4).to(dev, torch.float32).contiguous()
    assert pr.shape == gt.shape
    pts = p3ds.to(torch.float32).contiguous()
    f, p = pr.size(0), pts.size(0)
    add = torch.empty((f,), dtype=torch.float32, device=dev)
    adds = torch.empty((f,), dtype=torch.float32, device=dev)
    ws_bytes = int(lib.pvn3d_pose_add_adds_workspace_bytes(f, p))
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        rc = lib.pvn3d_pose_add_adds(ptr(pr), ptr(gt), f, ptr(pts), p, ptr(add), ptr(adds), ptr(ws), ws_bytes,
                                     torch.cuda.current_stream(dev).cuda_stream)
    check(rc, "pvn3d_pose_add_adds")
    ws.record_stream(torch.cuda.current_stream(dev))
    return add, adds


def cal_add_cuda(pred_RT, gt_RT, p3ds) -> torch.Tensor:
    """Basic_Utils.cal_add_cuda (basic_utils.py:617-623): 0-dim tensor"""
    return pose_add_adds(pred_RT, gt_RT, p3ds)[0][0]


def cal_adds_cuda(pred_RT, gt_RT, p3ds) -> torch.Tensor:
    """Basic_Utils.cal_adds_cuda (basic_utils.py:625-635): 0-dim tensor"""
    return pose_add_adds(pred_RT, gt_RT, p3ds)[1][0]


# --------------------------------------------------------------------------------------------------
# scoring a batch: TorchEval.eval_metric / eval_metric_lm, cal_auc, cal_lm_add (pvn3d_eval_utils.py:113-343)
# --------------------------------------------------------------------------------------------------
ABSENT_RULES = {"zeros": 0, "identity": 1}   # PVN3D_ADD_ABSENT_ZEROS / _IDENTITY


def pack_meshes(meshes) -> Tuple[np.ndarray, np.ndarray]:
    """{class id: [P,3]} (or a list indexed by class id, entry 0 ignored) -> (points [P_total,3] f32,
    mesh_off [n_cls+1] i32) with n_cls = largest id + 1.  Every class 1 .. n_cls-1 needs at least one point."""
    items = dict(meshes) if isinstance(meshes, dict) else dict(enumerate(meshes))
    items.pop(0, None)
    if not items:
        raise ValueError("pack_meshes: no class meshes")
    n_cls = max(int(c) for c in items) + 1
    pts, off = [np.zeros((0, 3), np.float32)], [0, 0]
    for c in range(1, n_cls):
        m = items.get(c)
        m = None if m is None else np.asarray(m.detach().cpu() if torch.is_tensor(m) else m, np.float32).reshape(-1, 3)
        if m is None or m.shape[0] == 0:
            raise ValueError(f"pack_meshes: class {c} has no mesh points")
        pts.append(m)
        off.append(off[-1] + m.shape[0])
    return np.ascontiguousarray(np.concatenate(pts, 0)), np.asarray(off, np.int32)


def scored_slots(cls_ids: np.ndarray, n_cls: int) -> np.ndarray:
    """[B,I] bool: the slots eval_metric scores -- those before the first class 0 of their frame (the `break` at
    pvn3d_eval_utils.py:118-119) whose class has a mesh (1 <= id < n_cls); frame_add_adds writes NaN elsewhere"""
    ids = np.asarray(cls_ids).reshape(np.shape(cls_ids)[0], -1)
    return (np.cumsum(ids == 0, axis=1) == 0) & (ids >= 1) & (ids < n_cls)


def frame_add_adds(poses: torch.Tensor, present: torch.Tensor, gt_rt: torch.Tensor, cls_ids: torch.Tensor,
                   meshes: torch.Tensor, mesh_off: np.ndarray, absent: str = "zeros") -> Tuple[torch.Tensor, torch.Tensor]:
    """ADD and ADD-S of every (frame, ground-truth slot) in one pair of launches, no host sync.
    poses [B,n_cls,3,4] f32 and present [B,n_cls] u8 (FramePoseSolver.solve / IcpRefiner.refine), gt_rt [B,I,3,4],
    cls_ids [B,I] or [B,I,1] (any integer dtype), meshes [P_total,3] f32 on the device with host offsets
    mesh_off [n_cls+1] (pack_meshes).  absent: "zeros" (YCB: a class the frame did not predict is scored with the
    zero pose) or "identity" (LineMOD).  -> (add [B,I], adds [B,I]) f32, NaN for the slots eval_metric skips."""
    if not (poses.is_cuda and meshes.is_cuda):
        raise RuntimeError("frame_add_adds (pvn3d_b200): CUDA tensors only -- no CPU fallback")
    if absent not in ABSENT_RULES:
        raise ValueError(f"absent must be one of {sorted(ABSENT_RULES)}, not {absent!r}")
    lib = _lib.load()
    dev = poses.device
    b, n_cls = poses.shape[:2]
    off = np.ascontiguousarray(mesh_off, dtype=np.int32)
    assert poses.shape[2:] == (3, 4) and off.shape == (n_cls + 1,), (tuple(poses.shape), off.shape)
    ps = poses.to(torch.float32).contiguous()
    pr = present.to(dev, torch.uint8).reshape(b, n_cls).contiguous()
    slots = gt_rt.shape[1]
    gt = gt_rt.to(dev, torch.float32).reshape(b, slots, 3, 4).contiguous()
    ids = cls_ids.to(dev, torch.int32).reshape(b, slots).contiguous()
    pts = meshes.to(torch.float32).contiguous()
    add = torch.empty((b, slots), dtype=torch.float32, device=dev)
    adds = torch.empty((b, slots), dtype=torch.float32, device=dev)
    max_p = int(np.diff(off)[1:].max()) if n_cls > 1 else 0
    ws_bytes = int(lib.pvn3d_frame_add_adds_workspace_bytes(b, slots, max_p))
    ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        rc = lib.pvn3d_frame_add_adds(ptr(ps), ptr(pr), n_cls, ptr(gt), ptr(ids), b, slots, ptr(pts),
                                      off.ctypes.data, ABSENT_RULES[absent], ptr(add), ptr(adds), ptr(ws), ws_bytes,
                                      torch.cuda.current_stream(dev).cuda_stream)
    check(rc, "pvn3d_frame_add_adds")
    ws.record_stream(torch.cuda.current_stream(dev))
    return add, adds


def voc_ap(rec: np.ndarray, prec: np.ndarray) -> float:
    """VOCap (basic_utils.py:32-44), vectorised: the running maximum of the precision over the finite recalls, and
    the precision taken at the FIRST element of each run of equal recalls"""
    idx = np.where(rec != np.inf)
    if len(idx[0]) == 0:
        return 0
    rec, prec = rec[idx], prec[idx]
    mrec = np.array([0.0] + list(rec) + [0.1])
    mpre = np.array([0.0] + list(prec) + [prec[-1]])
    m = prec.shape[0]
    mpre[:m] = np.maximum.accumulate(mpre[:m])       # the reference's loop runs over i = 1 .. m-1 only
    i = np.where(mrec[1:] != mrec[0:-1])[0] + 1
    return np.sum((mrec[i] - mrec[i - 1]) * mpre[i]) * 10


def cal_auc(add_dis, max_dis: float = 0.1) -> float:
    """Basic_Utils.cal_auc (basic_utils.py:597-604): distances > max_dis count as misses, the accuracy is the
    float32 cumulative count over n, area under it up to 0.1 m in percent (0 for an empty list)"""
    d = np.array(add_dis, dtype=np.float64)
    d[np.where(d > max_dis)] = np.inf
    d = np.sort(d)
    n = len(add_dis)
    acc = np.cumsum(np.ones((1, n)), dtype=np.float32) / n
    return voc_ap(d, acc) * 100


def append_distances(add_l: List[List[float]], adds_l: List[List[float]], add: np.ndarray, adds: np.ndarray,
                     cls_ids: np.ndarray) -> None:
    """append the scored slots of one batch ([B,I] host arrays) to the per-class lists as eval_pose_parallel does:
    frames in order, slots in order, each value under its class and under class 0"""
    for f, j in zip(*np.nonzero(scored_slots(cls_ids, len(add_l)))):
        c = int(cls_ids[f, j])
        for lst, v in ((add_l, add[f, j]), (adds_l, adds[f, j])):
            lst[c].append(float(v))
            lst[0].append(float(v))


def auc_table(add_l: List[List[float]], adds_l: List[List[float]], sym_cls_ids: Sequence[int]) -> Dict[str, object]:
    """TorchEval.cal_auc (pvn3d_eval_utils.py:249-281) without its prints and pickle: add_auc_lst / adds_auc_lst /
    add_s_auc_lst [n_cls] -- entry 0 over all objects (following PoseCNN); ADD(-S) is ADD-S for the classes in
    sym_cls_ids -- and their means over the classes 1 .. ("Average of all object")"""
    add_s = [[] for _ in add_l]
    for c in range(1, len(add_l)):
        add_s[c] = adds_l[c] if c in sym_cls_ids else add_l[c]
        add_s[0] = add_s[0] + add_s[c]
    out = {"add_auc_lst": [cal_auc(x) for x in add_l], "adds_auc_lst": [cal_auc(x) for x in adds_l],
           "add_s_auc_lst": [cal_auc(x) for x in add_s]}
    for k in ("add", "adds", "add_s"):
        out[f"{k}_auc_mean"] = np.mean(out[f"{k}_auc_lst"][1:])
    return out


def lm_accuracy(add_dis, adds_dis, diameter: float) -> Tuple[float, float]:
    """TorchEval.cal_lm_add's percentages of ADD and ADD-S below 0.1 diameter (diameter in metres, :314-317)"""
    d = diameter * 0.1
    return np.mean(np.array(add_dis) < d) * 100, np.mean(np.array(adds_dis) < d) * 100


class PoseEvaluator:
    """TorchEval's scoring on the device: per (frame, ground-truth slot) ADD and ADD-S in one launch per batch, the
    per-class distance lists and their AUCs as TorchEval.cal_auc / cal_lm_add compute them.

        ev = PoseEvaluator(meshes, sym_cls_ids=[13, 16, 19, 20, 21])         # YCB
        for batch in loader:
            poses, present, _, _ = solver.solve(...)
            ev.add_batch(poses, present, RTs, cls_ids)                          # no host sync
        add, adds = ev.distances()                                              # one device -> host read
        res = ev.auc()

    meshes: {class id: [P,3]} or a list indexed by class id (entry 0 ignored) -- every class 1 .. n_cls-1 needs
    points; n_cls = largest id + 1 must equal the pose table's second dimension.  sym_cls_ids: classes whose ADD(-S)
    is ADD-S.  diameters: {class id: diameter in metres} for lm_accuracy.  absent: "zeros" (YCB) or "identity"
    (LineMOD), the pose a class the frame did not predict is scored with."""

    def __init__(self, meshes, sym_cls_ids: Sequence[int] = (), diameters=None, absent: str = "zeros",
                 device="cuda"):
        if absent not in ABSENT_RULES:
            raise ValueError(f"absent must be one of {sorted(ABSENT_RULES)}, not {absent!r}")
        self.dev = torch.device(device)
        if self.dev.type != "cuda":
            raise RuntimeError("PoseEvaluator: CUDA only -- no CPU fallback")
        pts, self.mesh_off = pack_meshes(meshes)
        self.meshes = torch.from_numpy(pts).to(self.dev)
        self.n_cls = self.mesh_off.size - 1
        self.sym_cls_ids = [int(c) for c in sym_cls_ids]
        self.diameters = diameters
        self.absent = absent
        self.reset()

    def reset(self) -> None:
        """forget every batch scored so far"""
        self._pending: List[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = []
        self._add: List[List[float]] = [[] for _ in range(self.n_cls)]
        self._adds: List[List[float]] = [[] for _ in range(self.n_cls)]

    def add_batch(self, poses: torch.Tensor, present: torch.Tensor, gt_rt: torch.Tensor,
                  cls_ids: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """score one batch (see frame_add_adds) and keep the result; sync-free with device inputs.
        -> (add [B,I], adds [B,I]) on the device, NaN for the slots eval_metric skips"""
        if poses.shape[1] != self.n_cls:
            raise ValueError(f"pose table has {poses.shape[1]} classes, the meshes {self.n_cls}")
        add, adds = frame_add_adds(poses, present, gt_rt, cls_ids, self.meshes, self.mesh_off, self.absent)
        ids = cls_ids.to(self.dev, torch.int32).reshape(add.shape)
        self._pending.append((add, adds, ids))
        return add, adds

    def distances(self) -> Tuple[List[List[float]], List[List[float]]]:
        """(cls_add_dis, cls_adds_dis): per class id, the distances of every scored slot, class 0 holding all of
        them, in the order eval_pose_parallel appends them (batches, then frames, then slots).  One device -> host
        read for the batches added since the last call."""
        if self._pending:
            flat = torch.cat([torch.stack((a.reshape(-1), s.reshape(-1), c.reshape(-1).to(torch.float32)))
                              for a, s, c in self._pending], 1).cpu().numpy()
            shapes = [tuple(a.shape) for a, _, _ in self._pending]
            self._pending = []
            at = 0
            for b, i in shapes:
                a, d, c = (flat[k, at:at + b * i].reshape(b, i) for k in range(3))
                at += b * i
                append_distances(self._add, self._adds, a, d, c.astype(np.int64))
        return [list(x) for x in self._add], [list(x) for x in self._adds]

    def auc(self) -> Dict[str, object]:
        """TorchEval.cal_auc's numbers: add_auc_lst / adds_auc_lst / add_s_auc_lst [n_cls] (entry 0: all objects,
        following PoseCNN) and their means over the classes (entries 1 ..)"""
        return auc_table(*self.distances(), self.sym_cls_ids)

    def lm_accuracy(self, cls: int) -> Tuple[float, float]:
        """TorchEval.cal_lm_add's (ADD, ADD-S) < 0.1 diameter, in percent, of class `cls`"""
        if self.diameters is None:
            raise ValueError("lm_accuracy needs the class diameters")
        add, adds = self.distances()
        return lm_accuracy(add[cls], adds[cls], self.diameters[cls])
