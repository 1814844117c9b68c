"""Float64 restatements of get_item's target block and of lib/loss.py's FocalLoss / OFLoss (numpy and CPU torch, no GPU),
plus the wrong variants ("mutants") the goldens of tests/golden/train_cases.npz must tell apart:

    targets_ref   ycb_dataset.py:241-278: kps = kp_f32 . r^T + t and ctr likewise in float64; offset =
                  float32(float64(cld) - kp); the LAST meta slot of a class wins; labels in no slot stay zero
    focal_ref     FocalLoss(gamma): logpt = log_softmax(z)[t], pt = exp(logpt) detached; mean (or sum) of
                  -(1-pt)^gamma logpt; optional row mask (PVN3DLoss's ok frames)
    of_ref        OFLoss: [bs, n_kpts] = sum_{n,c} w |pred - targ| / (sum_n w + 1e-3), w = labels > 1e-8.  The
                  denominator counts each labelled point ONCE: the weight tensor lib/loss.py sums is [bs,n_kpts,n_pts,1]

MUTANTS: "first_slot_wins" (targets), "pt_not_detached" (focal), "den_3x" (OF: a denominator of 3x the count, as if w
were summed over the three coordinates too).
"""
from __future__ import annotations

import hashlib

import numpy as np
import torch

MUTANTS = ("first_slot_wins", "pt_not_detached", "den_3x")
ROW_STRIDE = 8       #: tests/golden/train_cases.npz keeps every ROW_STRIDE-th point of get_item's kp_targ_ofst


def digest(a) -> str:
    """SHA-256 of an array's dtype, shape and C-order bytes: how the goldens keep get_item's large outputs"""
    a = np.ascontiguousarray(a)
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return h.hexdigest()


def cld_rgb_nrm_of(pcld, rgb, choose):
    """get_item's cld_rgb_nrm [B,N,9] f32 with get_normal stubbed to zeros: (cld, rgb at choose, 0) -- rgb [B,3,H,W]
    (integer colours), choose [B,1,N] pixel indices"""
    b, n = np.shape(pcld)[:2]
    col = np.take_along_axis(np.asarray(rgb).reshape(b, 3, -1), np.asarray(choose).reshape(b, 1, n).repeat(3, 1), 2)
    return np.concatenate([np.asarray(pcld, np.float32), col.transpose(0, 2, 1).astype(np.float32),
                           np.zeros((b, n, 3), np.float32)], 2)


def targets_ref(pcld, labels, cls_ids, rts, kp_table, ctr_table, mutant=None):
    """pcld [B,N,3] f32, labels [B,N] int, cls_ids [B,S] int, rts [B,S,3,4] f64, kp_table [n_cls,K,3] f32,
    ctr_table [n_cls,3] f32 -> float32 (kp_targ [B,N,K,3], ctr_targ [B,N,3], kp3ds [B,S,K,3], ctr3ds [B,S,3])"""
    pcld = np.asarray(pcld, np.float32)
    b, n = labels.shape
    s = cls_ids.shape[1]
    n_cls, k = kp_table.shape[:2]
    kp_t = np.zeros((b, n, k, 3))
    ctr_t = np.zeros((b, n, 3))
    kp3 = np.zeros((b, s, k, 3))
    ctr3 = np.zeros((b, s, 3))
    for f in range(b):
        order = range(s - 1, -1, -1) if mutant == "first_slot_wins" else range(s)
        for i in order:
            c = int(cls_ids[f, i])
            if not 1 <= c < n_cls:
                continue
            r = np.asarray(rts[f, i, :, :3], np.float64)
            t = np.asarray(rts[f, i, :, 3], np.float64)
            kps = np.dot(np.asarray(kp_table[c], np.float32), r.T) + t
            ctr = np.dot(np.asarray(ctr_table[c], np.float32)[:, None].T, r.T)[0] + t
            kp3[f, i], ctr3[f, i] = kps, ctr
            m = np.where(labels[f] == c)[0]
            cld = pcld[f, m].astype(np.float64)
            ctr_t[f, m] = cld - ctr
            kp_t[f, m] = cld[:, None, :] - kps[None]
    return tuple(a.astype(np.float32) for a in (kp_t, ctr_t, kp3, ctr3))


def focal_ref(z, target, gamma, mean=True, row_mask=None, mutant=None):
    """float64 FocalLoss of z [M,C] against target [M] -> (loss, d loss / d z [M,C]).  A target outside [0, C) gives a
    NaN row.  row_mask [M] bool: rows left out (PVN3DLoss's ok = 0 frames); with no row left the loss is 0."""
    z = torch.as_tensor(np.asarray(z, np.float64)).clone().requires_grad_(True)
    t = torch.as_tensor(np.asarray(target, np.int64))
    c = z.shape[1]
    valid = (t >= 0) & (t < c)
    logp = torch.log_softmax(z, 1)
    logpt = logp.gather(1, torch.where(valid, t, 0)[:, None])[:, 0]
    logpt = torch.where(valid, logpt, torch.full_like(logpt, float("nan")))
    pt = logpt.exp() if mutant == "pt_not_detached" else logpt.detach().exp()
    rows = -1 * (1 - pt) ** gamma * logpt
    if row_mask is not None:
        rows = rows[torch.as_tensor(np.asarray(row_mask, bool))]
    if rows.numel() == 0:
        loss = (z * 0).sum()
    else:
        loss = rows.mean() if mean else rows.sum()
    loss.backward()
    return float(loss), z.grad.numpy()


def of_ref(pred, targ, labels, g=None, mutant=None):
    """float64 OFLoss: pred [bs,K,n,3], targ (viewed as [bs,n,K,3]), labels [bs,n] -> (loss [bs,K], d sum(g * loss) /
    d pred [bs,K,n,3]); g [bs,K] defaults to ones"""
    pred = torch.as_tensor(np.asarray(pred, np.float64)).clone().requires_grad_(True)
    bs, k, n, _ = pred.shape
    targ = torch.as_tensor(np.asarray(targ, np.float64)).reshape(bs, n, k, 3).permute(0, 2, 1, 3)
    w = torch.as_tensor(np.asarray(labels).reshape(bs, 1, n, 1) > 1e-8).float()
    s = (w * (pred - targ).abs()).sum((2, 3))
    cnt = w.sum((2, 3)) * (3 if mutant == "den_3x" else 1)
    loss = s / (cnt + 1e-3)        # w is float32 in lib/loss.py: its denominator is float32(count + 1e-3)
    gg = torch.ones(bs, k, dtype=torch.float64) if g is None else torch.as_tensor(np.asarray(g, np.float64))
    (loss * gg).sum().backward()
    return loss.detach().numpy(), pred.grad.numpy()


def pvn3d_loss_ref(kp, seg, ctr, kp_targ, ctr_targ, labels, ok=None, weights=(2.0, 1.0, 1.0), gamma=2.0):
    """PVN3DLoss in float64: (loss, parts [3], acc, d_kp, d_seg, d_ctr) for d loss"""
    b, k, n, _ = kp.shape
    lab = np.asarray(labels).reshape(b, n)
    mask = None if ok is None else np.repeat(np.asarray(ok).reshape(b) != 0, n)
    z = np.asarray(seg, np.float64).reshape(b * n, -1)
    focal, d_seg = focal_ref(z, lab.reshape(-1), gamma, row_mask=mask)
    kl, d_kp = of_ref(kp, kp_targ, lab, g=np.full((b, k), weights[1]))
    cl, d_ctr = of_ref(ctr, ctr_targ, lab, g=np.full((b, ctr.shape[1]), weights[2]))
    parts = np.array([focal, kl.sum(), cl.sum()])
    loss = weights[0] * parts[0] + weights[1] * parts[1] + weights[2] * parts[2]
    hit = np.argmax(z, 1) == lab.reshape(-1)
    m = len(hit) if mask is None else int(mask.sum())
    acc = (hit if mask is None else hit[mask]).sum() / m if m else 0.0
    return loss, parts, acc, d_kp, weights[0] * d_seg.reshape(np.shape(seg)), d_ctr
