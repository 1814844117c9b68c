"""Float64 restatements of get_item's target block and of lib/loss.py's FocalLoss / OFLoss (numpy and torch; the
loss functions run on whatever device their inputs are on, so the large edge cases can run their float64 reference on
the GPU), plus the wrong variants ("mutants") the goldens of tests/golden/train_cases.npz must tell apart:

    targets_ref   ycb_dataset.py:241-278: kps = kp_f32 . r^T + t and ctr likewise in float64; offset =
                  float32(float64(cld) - kp); the LAST meta slot of a class wins; labels in no slot stay zero
    focal_ref     FocalLoss(gamma): logpt = log_softmax(z)[t], pt = exp(logpt) detached; mean (or sum) of
                  -(1-pt)^gamma logpt; optional row mask (PVN3DLoss's ok frames)
    of_ref        OFLoss: [bs, n_kpts] = sum_{n,c} w |pred - targ| / (sum_n w + 1e-3), w = labels > 1e-8.  The
                  denominator counts each labelled point ONCE: the weight tensor lib/loss.py sums is [bs,n_kpts,n_pts,1]

    pvn3d_loss_t  PVN3DLoss: weights . (focal, sum OF kp, sum OF ctr) with an ok frame mask, and the gradient of
                  g_loss * loss + g_parts . parts

MUTANTS: "first_slot_wins" (targets), "pt_not_detached" (focal), "den_3x" (OF: a denominator of 3x the count, as if w
were summed over the three coordinates too).  The edge cases (tests/train_edge_cases.py) add "gamma_rounded",
"tail_dropped" and "ok_ignored" (focal), "nhwc" (nchw_rows), "den_no_eps" and "tail_dropped" (OF), and
"g_parts_ignored" (PVN3DLoss).
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


def _f64(x, device=None):
    t = torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x)
    return t.to(device=device if device is not None else t.device, dtype=torch.float64)


def nchw_rows(z, mutant=None):
    """FocalLoss's rows of an [N,C,*] input: [N * prod(*), C] with row (n, i) = z[n, :, i], as lib/loss.py's
    view / transpose / view makes them; a 2-D input is its own rows.  Mutant "nhwc": the same memory read as if
    each row's C values were contiguous."""
    z = torch.as_tensor(z)
    if z.dim() == 2:
        return z
    n, c = z.shape[:2]
    if mutant == "nhwc":
        return z.reshape(-1, c)
    return z.reshape(n, c, -1).transpose(1, 2).reshape(-1, c)


def focal_t(z, target, gamma, mean=True, row_mask=None, g=1.0, mutant=None, tile=128):
    """float64 FocalLoss on torch tensors, on z's device: z [M,C], target [M] -> (loss [], d (g loss) / d z [M,C]).
    A target outside [0, C) gives a NaN row.  row_mask [M] bool: rows left out of the sum and the divisor
    (PVN3DLoss's ok = 0 frames); with no row left the loss is 0.
    Mutants: "pt_not_detached", "gamma_rounded" (gamma to the nearest integer), "tail_dropped" (the rows after the
    last full tile of `tile` rows add nothing, the divisor stays M), "ok_ignored" (row_mask is not applied)."""
    z = _f64(z).clone().requires_grad_(True)
    t = torch.as_tensor(np.asarray(target) if not torch.is_tensor(target) else target).to(z.device, torch.int64)
    m, c = z.shape
    if mutant == "gamma_rounded":
        gamma = float(round(gamma))
    valid = (t >= 0) & (t < c)
    logp = torch.log_softmax(z, 1)
    logpt = logp.gather(1, torch.where(valid, t, 0)[:, None])[:, 0]
    logpt = torch.where(valid, logpt, torch.full_like(logpt, float("nan")))
    pt = logpt.exp() if mutant == "pt_not_detached" else logpt.detach().exp()
    rows = -1 * (1 - pt) ** gamma * logpt
    if mutant == "tail_dropped":
        rows = torch.where(torch.arange(m, device=z.device) < m // tile * tile, rows, torch.zeros_like(rows))
    if row_mask is not None and mutant != "ok_ignored":
        rows = rows[torch.as_tensor(np.asarray(row_mask, bool) if not torch.is_tensor(row_mask) else row_mask,
                                    device=z.device)]
    if rows.numel() == 0:
        loss = (z * 0).sum()
    else:
        loss = rows.mean() if mean else rows.sum()
    (loss * g).backward()
    return loss.detach(), z.grad


def focal_ref(z, target, gamma, mean=True, row_mask=None, mutant=None):
    """focal_t with numpy in and out: (loss float, d loss / d z [M,C])"""
    loss, grad = focal_t(z, target, gamma, mean=mean, row_mask=row_mask, mutant=mutant)
    return float(loss), grad.cpu().numpy()


def of_t(pred, targ, labels, g=None, mutant=None, tile=128):
    """float64 OFLoss on torch tensors, on pred's device: pred [bs,K,n,3], targ (viewed as [bs,n,K,3]), labels
    [bs,n] (integer, or float with w = labels > 1e-8) -> (loss [bs,K], d sum(g * loss) / d pred [bs,K,n,3]); g [bs,K]
    defaults to ones.  Mutants: "den_3x" (three times the count), "den_no_eps" (the count alone), "tail_dropped"
    (each frame's points after its last full tile of `tile` points are left out)."""
    pred = _f64(pred).clone().requires_grad_(True)
    dev = pred.device
    bs, k, n, _ = pred.shape
    targ = _f64(targ, dev).reshape(bs, n, k, 3).permute(0, 2, 1, 3)
    lab = torch.as_tensor(np.asarray(labels) if not torch.is_tensor(labels) else labels).to(dev).reshape(bs, 1, n, 1)
    w = (lab > 1e-8).float()
    if mutant == "tail_dropped":
        w = w * (torch.arange(n, device=dev) < n // tile * tile).reshape(1, 1, n, 1)
    s = (w * (pred - targ).abs()).sum((2, 3))
    cnt = w.sum((2, 3)) * (3 if mutant == "den_3x" else 1)
    # w is float32 in lib/loss.py: its denominator is float32(count + 1e-3)
    loss = s / (cnt if mutant == "den_no_eps" else cnt + 1e-3)
    gg = torch.ones(bs, k, dtype=torch.float64, device=dev) if g is None else _f64(g, dev).expand(bs, k)
    (loss * gg).sum().backward()
    return loss.detach(), pred.grad


def of_ref(pred, targ, labels, g=None, mutant=None):
    """of_t with numpy in and out"""
    loss, grad = of_t(pred, targ, labels, g=g, mutant=mutant)
    return loss.cpu().numpy(), grad.cpu().numpy()


def pvn3d_loss_t(kp, seg, ctr, kp_targ, ctr_targ, labels, ok=None, weights=(2.0, 1.0, 1.0), gamma=2.0, g_loss=1.0,
                 g_parts=(0.0, 0.0, 0.0), mutant=None):
    """PVN3DLoss in float64 on torch tensors, on kp's device: dict(loss, parts [3], acc, d_kp, d_seg, d_ctr) with the
    gradients of g_loss * loss + g_parts . parts, where loss = weights . parts and parts = (focal over the rows of ok
    frames, sum of the kp OFLoss, sum of the ctr OFLoss).  Mutants: "ok_ignored", "g_parts_ignored"."""
    dev = torch.as_tensor(kp).device
    b, k, n, _ = kp.shape
    lab = torch.as_tensor(np.asarray(labels) if not torch.is_tensor(labels) else labels).to(dev).reshape(b, n)
    mask = None
    if ok is not None:
        okt = torch.as_tensor(np.asarray(ok) if not torch.is_tensor(ok) else ok).to(dev).reshape(b) != 0
        mask = okt.repeat_interleave(n)
    gp = (0.0, 0.0, 0.0) if mutant == "g_parts_ignored" else tuple(float(v) for v in g_parts)
    gs = [g_loss * w + v for w, v in zip(weights, gp)]      # d (g_loss loss + g_parts . parts) / d parts
    z = _f64(seg, dev).reshape(b * n, -1)
    focal, d_seg = focal_t(z, lab.reshape(-1), gamma, row_mask=mask, g=gs[0],
                           mutant="ok_ignored" if mutant == "ok_ignored" else None)
    kl, d_kp = of_t(kp, kp_targ, lab, g=gs[1])
    cl, d_ctr = of_t(ctr, ctr_targ, lab, g=gs[2])
    parts = torch.stack([focal, kl.sum(), cl.sum()])
    loss = weights[0] * parts[0] + weights[1] * parts[1] + weights[2] * parts[2]
    hit = (torch.argmax(z, 1) == lab.reshape(-1)).double()
    if mask is not None and mutant != "ok_ignored":
        hit = hit[mask]
    acc = hit.mean() if hit.numel() else torch.zeros((), dtype=torch.float64, device=dev)
    return dict(loss=loss, parts=parts, acc=acc, d_kp=d_kp, d_seg=d_seg.reshape(np.shape(seg)), d_ctr=d_ctr)


def pvn3d_loss_ref(kp, seg, ctr, kp_targ, ctr_targ, labels, ok=None, weights=(2.0, 1.0, 1.0), gamma=2.0):
    """pvn3d_loss_t with numpy in and out: (loss, parts [3], acc, d_kp, d_seg, d_ctr) for d loss"""
    r = pvn3d_loss_t(kp, seg, ctr, kp_targ, ctr_targ, labels, ok, weights, gamma)
    return (float(r["loss"]), r["parts"].numpy(), float(r["acc"]), r["d_kp"].numpy(), r["d_seg"].numpy(),
            r["d_ctr"].numpy())


def raw_frames(b: int, h: int = 480, w: int = 640, seed: int = 0, sparse=()):
    """raw frames for train_utils.train_batch: depth (mm) of a curved background with four objects (classes 1, 4, 9, 4)
    0.5 m in front of it, their label image, a YCB camera, random colours and four poses -> (depth, K, cam_scale, rgb,
    label, cls_ids, RTs) as numpy arrays.  The frames listed in `sparse` keep only 300 valid depth pixels, too few for
    get_item (FrameInputBuilder's ok = 0); the random draws do not depend on `sparse`."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    depth = np.zeros((b, h, w), np.float32)
    label = np.zeros((b, h, w), np.int32)
    for f in range(b):
        depth[f] = 9000 + 500 * np.sin(xx / (60.0 + f)) + 300 * np.cos(yy / 50.0)
        for c in (1, 4, 9, 4):
            y0, x0 = rng.integers(0, h - 120), rng.integers(0, w - 150)
            label[f, y0:y0 + 120, x0:x0 + 150] = c
            depth[f, y0:y0 + 120, x0:x0 + 150] -= 500
    for f in sparse:
        depth[f] = 0
        depth[f, 100:110, 100:130] = 8000
    K = np.tile(np.float32([[1066.778, 0, 312.9869], [0, 1067.487, 241.3109], [0, 0, 1]]), (b, 1, 1))
    rgb = rng.integers(0, 256, (b, 3, h, w), dtype=np.uint8)
    ids = np.zeros((b, 22), np.int64)
    ids[:, :4] = [1, 4, 9, 4]
    rts = np.zeros((b, 22, 3, 4))
    for f in range(b):
        for i in range(4):
            q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
            rts[f, i] = np.concatenate([q, rng.normal(0, 0.2, (3, 1)) + [[0], [0], [0.9]]], 1)
    return depth, K, np.full(b, 10000.0, np.float32), rgb, label, ids, rts
