"""float64 restatement of TorchEval's per-slot scoring (eval_metric / eval_metric_lm, pvn3d_eval_utils.py:113-137,
204-220) and of the AUC bookkeeping of cal_auc (basic_utils.py:32-44,597-604), with the wrong variants a kernel or a
port could plausibly produce.  The tests use it as the brute-force reference of pvn3d_frame_add_adds and to show that
the recorded goldens (tests/golden/eval_cases.npz) tell every variant apart.

Mutants (`mutant=`):
  "absent_swapped"   the other absent rule: identity under YCB, zeros under LineMOD
  "past_zero"        slots after the first class 0 of a frame scored too
  "cls_off_by_one"   the mesh of class c-1 used for class c (class 1 keeps its own)
  "frame_shift"      the poses of frame b+1 (mod B) used for frame b
  "sym_swapped"      ADD(-S) takes ADD for the symmetric classes and ADD-S for the rest
  "tie_last"         VOCap takes the precision at the LAST element of each run of equal distances
"""
from __future__ import annotations

import numpy as np

IDENTITY = np.eye(4)[:3]


def slot_mask(cls_ids, n_cls, mutant=None):
    ids = np.asarray(cls_ids).reshape(np.shape(cls_ids)[0], -1)
    before_zero = np.cumsum(ids == 0, axis=1) == 0
    if mutant == "past_zero":
        before_zero = np.ones_like(before_zero)
    return before_zero & (ids >= 1) & (ids < n_cls)


def add_adds_f64(pred, gt, pts):
    """ADD and ADD-S of one pose pair over one mesh, in float64"""
    pts = np.asarray(pts, np.float64)
    pd = pts @ np.asarray(pred, np.float64)[:, :3].T + np.asarray(pred, np.float64)[:, 3]
    g = pts @ np.asarray(gt, np.float64)[:, :3].T + np.asarray(gt, np.float64)[:, 3]
    add = np.linalg.norm(pd - g, axis=1).mean()
    d2 = ((g[:, None, :] - pd[None, :, :]) ** 2).sum(-1)
    return add, np.sqrt(d2.min(1)).mean()


def frame_scores(poses, present, gt_rt, cls_ids, meshes, absent, mutant=None):
    """[B,I] float64 ADD and ADD-S of every slot (NaN where eval_metric scores nothing).  meshes: list indexed by
    class id; absent: "zeros" | "identity"."""
    poses = np.asarray(poses, np.float64)
    b, n_cls = poses.shape[:2]
    ids = np.asarray(cls_ids).reshape(b, -1).astype(np.int64)
    gt = np.asarray(gt_rt, np.float64).reshape(b, ids.shape[1], 3, 4)
    if mutant == "absent_swapped":
        absent = "identity" if absent == "zeros" else "zeros"
    scored = slot_mask(ids, n_cls, mutant)
    add = np.full(ids.shape, np.nan)
    adds = np.full(ids.shape, np.nan)
    for f in range(b):
        pf = (f + 1) % b if mutant == "frame_shift" else f
        for i in range(ids.shape[1]):
            if not scored[f, i]:
                continue
            c = int(ids[f, i])
            if present[pf][c]:
                pred = poses[pf, c]
            else:
                pred = IDENTITY if absent == "identity" else np.zeros((3, 4))
            mesh = meshes[c - 1] if (mutant == "cls_off_by_one" and c > 1) else meshes[c]
            add[f, i], adds[f, i] = add_adds_f64(pred, gt[f, i], mesh)
    return add, adds


def voc_ap(rec, prec, mutant=None):
    """VOCap (basic_utils.py:32-44) as a loop"""
    rec, prec = np.asarray(rec), np.asarray(prec)
    keep = rec != np.inf
    if not keep.any():
        return 0
    rec, prec = rec[keep], prec[keep]
    mrec = np.concatenate([[0.0], rec, [0.1]])
    mpre = np.concatenate([[0.0], prec.astype(np.float64), [prec[-1]]])
    for i in range(1, prec.shape[0]):
        mpre[i] = max(mpre[i], mpre[i - 1])
    if mutant == "tie_last":
        i = np.where(mrec[1:] != mrec[:-1])[0] + 1
        # the last element of the run that ends at mrec[i]: the step before the next change
        ends = np.concatenate([i[1:] - 1, [len(mrec) - 1]])
        return np.sum((mrec[i] - mrec[i - 1]) * mpre[np.minimum(np.maximum(ends, i), len(mpre) - 1)]) * 10
    i = np.where(mrec[1:] != mrec[:-1])[0] + 1
    return np.sum((mrec[i] - mrec[i - 1]) * mpre[i]) * 10


def cal_auc(dis, max_dis=0.1, mutant=None):
    d = np.array(dis, dtype=np.float64)
    d[d > max_dis] = np.inf
    d = np.sort(d)
    n = len(dis)
    acc = np.cumsum(np.ones((1, n)), dtype=np.float32) / n
    return voc_ap(d, acc, mutant) * 100


def add_s_lists(add, adds, sym_cls_ids, mutant=None):
    """TorchEval.cal_auc's cls_add_s_dis: ADD-S for the symmetric classes, ADD for the rest; entry 0 their
    concatenation in class order"""
    out = [[] for _ in add]
    for c in range(1, len(add)):
        sym = c in sym_cls_ids
        if mutant == "sym_swapped":
            sym = not sym
        out[c] = list(adds[c] if sym else add[c])
        out[0] += out[c]
    return out
