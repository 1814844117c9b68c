"""The inputs and bounds of tests/test_train_edges_gpu.py: csrc/train.cu's targets and loss kernels at the edges of
their tiling, their shared-memory footprints and their integer inputs, with the mutants each bound must reject
(tests/train_ref.py).  tests/test_train_edges_host.py checks, without a GPU, that the builders hit those edges and
that every bound tells each mutant from the float64 reference.  The bounds are derived in the docstring of
tests/test_train_edges_gpu.py.

Shared-memory footprints, from the kernels' constants (train.cu):
  * the loss kernels take kLossTile = TILE rows or points per block;
  * a focal block stages its logits as C columns of TILE + 1 floats: seg_smem(C) = C * 129 * 4 B;
  * an OF block stages [TILE, K, 3] targets and TILE weights: of_smem(K) = 128 * (3K + 1) * 4 B;
  * train_loss_partials_kernel also holds STATIC_SMEM = 784 B of static shared memory (s_red[4 warps * 48], s_cnt[4];
    ptxas -v reports the same), and without cudaFuncAttributeMaxDynamicSharedMemorySize a launch may use
    SMEM_LIMIT = 48 KB of static and dynamic memory together: NO_OPT_IN_DYNAMIC = 48,368 B of dynamic memory.
So C = 94 (48,504 B) and C = 95 (49,020 B) fit under 48 KB but not beside the static arrays; C = 96 and K = 32 are
over 48 KB; K = 31 (48,128 B) fits either way.  No K lies between the two limits.
"""
import numpy as np
import torch

F32 = np.float32
U = 2.0 ** -24                     #: float32 unit roundoff

TILE = 128                         #: kLossTile: logits rows / points per loss block
WARPS = TILE // 32                 #: kLossWarps
KP_MAX = 48                        #: kLossMaxKp
C_MAX = 128                        #: kLossMaxClasses
STATIC_SMEM = WARPS * KP_MAX * 4 + WARPS * 4      #: s_red (float) + s_cnt (int) of train_loss_partials_kernel
SMEM_LIMIT = 48 * 1024             #: static + dynamic shared memory of a launch without the opt-in
NO_OPT_IN_DYNAMIC = SMEM_LIMIT - STATIC_SMEM
TGT_THREADS = 256                  #: kTgtThreads: points per block of train_targets_kernel
TGT_MAX_SMEM = 48 * 1024           #: kTgtMaxSmem (train_targets_kernel has no static shared memory)


def seg_smem(c):
    return c * (TILE + 1) * 4


def of_smem(k):
    return TILE * (3 * k + 1) * 4


def tgt_smem(s, k, n_cls):
    """train_targets_kernel: the slots' K keypoints and centre in float64, the label -> slot map and the tile's slots"""
    return s * (k + 1) * 3 * 8 + (n_cls + TGT_THREADS) * 4


# ---- FocalLoss --------------------------------------------------------------------------------------------------
FOCAL_M = (1, TILE - 1, TILE + 1, 320 * TILE + 1)
FOCAL_C = (1, 2, 31, 94, 95, 96, 127, 128)
GAMMAS = (0.0, 0.5, 1.0, 1.5, 2.0, 3.0)
LARGE_M = (1 << 24) + 3            #: not a float32 integer; 131,073 blocks of partials
FRESH_C = (94, 95, 96)
FRESH_K = (31, 32)


def focal_rows(m, c, seed):
    """logits [m, c] f32 (scale 3, a few rows far apart and a few exactly tied) and targets [m] int64 in [0, c)"""
    rng = np.random.default_rng(seed)
    z = (rng.normal(0, 3, (m, c))).astype(F32)
    t = rng.integers(0, c, m)
    if m > 8:
        z[1] *= 8                                   # one confident row per case, and one tie
        z[2] = z[2, 0]
    return z, t


# N,C,H,W shapes: each HW either crosses a 128-row tile boundary inside an image or puts several images in one tile
NCHW_HW = {1: (1, 1), 7: (1, 7), 100: (10, 10), 129: (3, 43), 1000: (25, 40), 1200: (30, 40)}
NCHW_N = (1, 3, 5)
NCHW_SHAPES = [(n, (3, 22, 31)[i % 3], h, w) for i, (n, (h, w)) in
               enumerate((n, hw) for hw in NCHW_HW.values() for n in NCHW_N)]
NCHW_SHAPES += [(3, 22, 77), (2, 5, 3, 5, 7)]       # [N, C, L] and a 5-D input


def nchw_case(shape, seed):
    """logits of `shape` (f32) and targets [N, *] (int64)"""
    rng = np.random.default_rng(seed)
    z = rng.normal(0, 2, shape).astype(F32)
    t = rng.integers(0, shape[1], (shape[0],) + tuple(shape[2:]))
    return z, t


def tile_images(rows_per_image, rows):
    """for each TILE-row tile of `rows` rows, how many images (blocks of rows_per_image rows) it holds rows of"""
    starts = np.arange(0, rows, TILE)
    ends = np.minimum(starts + TILE, rows) - 1
    return ends // rows_per_image - starts // rows_per_image + 1


# ---- OFLoss -----------------------------------------------------------------------------------------------------
OF_N = (1, TILE - 1, TILE, TILE + 1, 96 * TILE - 1, 96 * TILE + 1)
OF_K = (1, 8, 31, 32, 47, 48)
OF_B = (1, 5)


def of_case(b, n, k, seed):
    """pred [b,K,n,3], targ [b,n,K,3] f32, labels [b,n] int64.  With b > 1, frame 0 has no labelled point and frame
    b-1 has every point labelled; the other frames label about 40 % of their points, the last point always."""
    rng = np.random.default_rng(seed)
    pred = (rng.normal(0, 0.1, (b, k, n, 3))).astype(F32)
    targ = (rng.normal(0, 0.1, (b, n, k, 3))).astype(F32)
    lab = np.where(rng.random((b, n)) < 0.4, rng.integers(1, 22, (b, n)), 0)
    lab[:, -1] = 7                                  # the ragged tail holds a labelled point
    if b > 1:
        lab[0] = 0
        lab[-1] = rng.integers(1, 22, n)
    return pred, targ, lab.astype(np.int64)


FLOAT_LABELS = (0.0, 1e-9, 2e-8, 1.0, 0.5)       #: around lib/loss.py's `labels > 1e-8` cut


def of_nonfinite_case(seed):
    """pred with NaN, +inf and -inf at unlabelled points of frame 0 (keypoints 0, 1, 2), float32 labels around
    the 1e-8 cut; frame 1 stays finite"""
    b, n, k = 2, 3 * TILE + 5, 4
    rng = np.random.default_rng(seed)
    pred = (rng.normal(0, 0.1, (b, k, n, 3))).astype(F32)
    targ = (rng.normal(0, 0.1, (b, n, k, 3))).astype(F32)
    lab = np.asarray(FLOAT_LABELS, F32)[rng.integers(0, len(FLOAT_LABELS), (b, n))]
    lab[:, :3] = (0, 1e-9, 2e-8)
    pred[0, 0, 0, 1] = np.nan                       # label 0
    pred[0, 1, 1, 0] = np.inf                       # label 1e-9: below the cut
    pred[0, 2, TILE + 1, 2] = -np.inf
    lab[0, TILE + 1] = 0
    return pred, targ, lab


# ---- PVN3DLoss --------------------------------------------------------------------------------------------------
PVN_B, PVN_N = 5, 96 * TILE - 1                    #: 12287 points: every frame after the first starts mid-tile
PVN_OK = (1, 0, 1, 1, 0)
PVN_C = (22, 96, 128)
PVN_K = (8, 32, 48)
PVN_WEIGHTS = (0.5, 3.0, 0.0)
PVN_GAMMA = 1.5
# backward through: loss only, parts only, a * loss + v . parts, and parts[1] alone (the focal and centre terms get
# no gradient: their outputs carry none)
PVN_GRADS = {"loss": (1.0, (0.0, 0.0, 0.0)), "parts": (0.0, (0.75, 0.5, 2.0)), "both": (1.25, (0.5, 0.25, 3.0)),
             "kp_part": (0.0, (0.0, 1.0, 0.0))}


def pvn3d_case(b, n, c, k, seed):
    """(kp [b,K,n,3], seg [b,n,C], ctr [b,1,n,3], kp_targ [b,n,K,3], ctr_targ [b,n,3]) f32, labels [b,n] int64 in
    [0, C) with about 40 % foreground, in every frame (the ok = 0 frames too, so ignoring ok changes the loss)"""
    rng = np.random.default_rng(seed)
    seg = (rng.normal(0, 3, (b, n, c))).astype(F32)
    lab = np.where(rng.random((b, n)) < 0.4, rng.integers(0, c, (b, n)), 0).astype(np.int64)
    kp = (rng.normal(0, 0.1, (b, k, n, 3))).astype(F32)
    ctr = (rng.normal(0, 0.1, (b, 1, n, 3))).astype(F32)
    kt = (rng.normal(0, 0.1, (b, n, k, 3))).astype(F32)
    ct = (rng.normal(0, 0.1, (b, n, 3))).astype(F32)
    return kp, seg, ctr, kt, ct, lab


# ---- targets ----------------------------------------------------------------------------------------------------
WIDE_IDS = ((1 << 32) + 1, (1 << 32) + 5, -(1 << 32) + 3, 1 << 62, -(1 << 63), (1 << 63) - 1)
TGT_N = (1, TGT_THREADS - 1, TGT_THREADS + 1)
TGT_K = (1, 48)
#: S = 30 slots of K = 48 and n_cls = 3212 classes fill train_targets_kernel's shared memory exactly
TGT_FULL = (30, 48, 12032 - 6 * 30 * 49)
TGT_MANY_FRAMES = 65535                            #: grid.y's limit, one point per frame


def _poses(rng, b, s):
    rts = np.zeros((b, s, 3, 4))
    q, _ = np.linalg.qr(rng.normal(size=(b * s, 3, 3)))
    rts[..., :3] = q.reshape(b, s, 3, 3)
    rts[..., 3] = rng.normal(0, 0.3, (b, s, 3))
    return rts


def targets_case(b, n, s, k, n_cls, seed, wide=False):
    """(pcld [b,n,3] f32, labels [b,n] int64, cls_ids [b,s] int64, rts [b,s,3,4] f64, kp_table [n_cls,K,3],
    ctr_table [n_cls,3] f32).  wide: labels and ids include WIDE_IDS, whose int32 truncation is a real class
    (2**32 + 1 -> 1, 2**32 + 5 -> 5, -2**32 + 3 -> 3) or an id that wraps (2**62 -> 0, -2**63 -> 0, 2**63 - 1 -> -1)"""
    rng = np.random.default_rng(seed)
    kp = rng.normal(0, 0.05, (n_cls, k, 3)).astype(F32)
    ctr = rng.normal(0, 0.02, (n_cls, 3)).astype(F32)
    pcld = (rng.normal(0, 0.3, (b, n, 3)) + [0, 0, 1]).astype(F32)
    labels = rng.integers(0, min(n_cls, 8), (b, n)).astype(np.int64)
    ids = np.zeros((b, s), np.int64)
    ids[:, :min(s, 7)] = np.arange(1, min(s, 7) + 1) % n_cls
    if s == 1:
        ids[:, 0] = rng.integers(1, n_cls, b)
        labels[:] = np.where(rng.random((b, n)) < 0.7, ids[:, :1], labels)
    if wide:
        w = np.asarray(WIDE_IDS, np.int64)
        labels.reshape(-1)[:len(w)] = w
        labels.reshape(-1)[-len(w):] = w[::-1]
        ids[:, -1] = w[np.arange(b) % len(w)]
        ids[0, 0] = w[1]                            # 2**32 + 5 in slot 0 of frame 0 (truncates to class 5)
    return pcld, labels, ids, _poses(rng, b, s), kp, ctr


# ---- bounds (derived in tests/test_train_edges_gpu.py) ------------------------------------------------------------
def focal_bounds(z, t, gamma, ref_grad, mean=True, row_mask=None, g=1.0):
    """(bound on |loss - ref|, bound [M,C] on |grad - ref grad|) of FocalLoss on logits z [M,C] (torch, any device)
    against targets t [M] in [0, C), for the gradient of g * loss"""
    z = torch.as_tensor(z).double()
    t = torch.as_tensor(t).to(z.device, torch.int64)
    c = z.shape[1]
    logpt = torch.log_softmax(z, 1).gather(1, t[:, None])[:, 0]
    a = logpt.abs()
    row = (1 - logpt.exp()) ** gamma * a
    e = (1 + gamma) * (4 * a + 2 * c + 16) * U
    if row_mask is not None:
        keep = torch.as_tensor(row_mask, device=z.device)
        e, row = torch.where(keep, e, 0.0), torch.where(keep, row, 0.0)
        m = max(int(keep.sum()), 1)
    else:
        m = z.shape[0]
    div = m if mean else 1
    lb = 2 * (((1 + a) * e).sum() + 12 * U * row.sum()) / div
    gb = 2 * abs(g) / div * e[:, None] + 8 * U * torch.as_tensor(ref_grad).abs()
    return float(lb), gb


def of_bounds(pred, targ, labels, ref_loss, ref_grad):
    """(bound [b,K] on |loss - ref|, bound on |grad - ref grad|) of OFLoss; pred [b,K,n,3], targ viewed as [b,n,K,3],
    labels [b,n] (torch, any device).  The gradient bound assumes g_loss, g_parts and g_kp do not cancel."""
    pred = torch.as_tensor(pred).double()
    b, k, n, _ = pred.shape
    targ = torch.as_tensor(targ).to(pred.device).double().reshape(b, n, k, 3).permute(0, 2, 1, 3)
    w = (torch.as_tensor(labels).to(pred.device).reshape(b, 1, n, 1) > 1e-8).double()
    s = torch.nan_to_num((w * (pred - targ).abs()).sum((2, 3)), nan=0.0, posinf=0.0)
    den = (w.sum((2, 3)).float() + 1e-3).double()
    lb = 2 * (11 * U * s / den + 3 * U * torch.nan_to_num(torch.as_tensor(ref_loss), nan=0.0).abs())
    gb = 6 * U * torch.nan_to_num(torch.as_tensor(ref_grad), nan=0.0).abs()
    return lb, gb


def sum_bound(values, bounds):
    """bound on a float32 sequential sum of float32 values, each within its bound of the reference"""
    values = torch.as_tensor(values).double()
    return float(torch.as_tensor(bounds).sum() + 2 * values.numel() * U * values.abs().sum())


def exceeds(got, want, bound):
    """True where |got - want| > bound (NaN in exactly one of got, want counts as exceeding; NaN in both does not)"""
    got, want = torch.as_tensor(got).double(), torch.as_tensor(want).double().to(torch.as_tensor(got).device)
    bound = torch.as_tensor(bound, dtype=torch.float64, device=got.device)
    both_nan = torch.isnan(got) & torch.isnan(want)
    return ~both_nan & ~((got - want).abs() <= bound)
