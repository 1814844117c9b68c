"""numpy restatement of ip_basic's fill_in_multiscale as Basic_Utils.fill_missing calls it (max_depth 3,
extrapolate False, blur 'bilateral'), stage by stage, for checking pvn3d_depth_fill.  No OpenCV: the
morphology, the median and cv2.bilateralFilter's float32 algorithm are written out here.

Steps 1-9 are float32 comparisons, selections and single float32 operations, so this module and the kernel
agree bit for bit there.  The bilateral filter computes every per-tap weight in float32 exactly as the
kernel does and accumulates in float64; the kernel accumulates in float32 (include/pvn3d_b200.h states the
bound).

`mutant=` selects a deliberately wrong variant, for tests that show a comparison can tell the difference:
  "median_reflect"   the median with a reflect-101 border instead of replicate
  "dilate_zero"      dilations that count outside pixels as 0 instead of ignoring them
  "loop_le"          `<= 0.01` instead of `< 0.01` in the six fill iterations
  "top1_loop"        top1 instead of top2 in the fill iterations and in V
  "five_iters"       five fill iterations instead of six
  "v_after_median"   V taken from the image after the median
  "minmax_valid"     the bilateral's min/max over the V pixels only
"""
from __future__ import annotations

import math

import numpy as np

MAX_DEPTH = np.float32(3.0)
T = np.float32(0.01)
F32 = np.float32
FLT_EPSILON = float(np.finfo(np.float32).eps)
EXP_BINS = 1 << 12
MUTANTS = ("median_reflect", "dilate_zero", "loop_le", "top1_loop", "five_iters", "v_after_median",
           "minmax_valid")


def _cross(n):
    k = np.zeros((n, n), bool)
    k[n // 2, :] = k[:, n // 2] = True
    return k


CROSS_3, CROSS_5, CROSS_7 = _cross(3), _cross(5), _cross(7)
FULL_5, FULL_9 = np.ones((5, 5), bool), np.ones((9, 9), bool)


def _window(img, kernel, pad_mode, pad_value=None):
    """[k, H, W]: img shifted by every offset of `kernel` (a boolean square mask)"""
    r = kernel.shape[0] // 2
    h, w = img.shape
    if pad_mode == "constant":
        p = np.pad(img, r, mode="constant", constant_values=pad_value)
    else:
        p = np.pad(img, r, mode=pad_mode)
    return np.stack([p[dy:dy + h, dx:dx + w] for dy, dx in zip(*np.nonzero(kernel))])


def dilate(img, kernel, border=-np.inf):
    """cv2.dilate: the window maximum; outside pixels are ignored (border -inf)"""
    return _window(img, kernel, "constant", F32(border)).max(0)


def erode(img, kernel):
    """cv2.erode: the window minimum; outside pixels are ignored (border +inf)"""
    return _window(img, kernel, "constant", F32(np.inf)).min(0)


def median5(img, mode="edge"):
    """cv2.medianBlur(img, 5) on float32: the 13th of the 25 window values, edge replicated"""
    return np.sort(_window(img, FULL_5, mode), axis=0)[12]


def top_rows(s):
    """per column, the first row with s > 0.01 (np.argmax: 0 when there is none)"""
    return np.argmax(s > T, axis=0)


def _under(top, h):
    return np.arange(h)[:, None] >= top[None, :]


def space_taps(radius=2, sigma_space=2.0):
    """cv2.bilateralFilter's taps in its order: (dy, dx, weight f32) for every offset with sqrt(dy^2 + dx^2)
    <= radius, rows outer, columns inner"""
    coeff = -0.5 / (sigma_space * sigma_space)
    taps = []
    for i in range(-radius, radius + 1):
        for j in range(-radius, radius + 1):
            r = math.sqrt(float(i * i + j * j))
            if r > radius:
                continue
            taps.append((i, j, F32(math.exp(r * r * coeff))))
    return taps


def bilateral_lut(vmin, vmax, sigma_color=0.5):
    """(scale_index f32, lut [4098] f32) of cv2's float32 bilateral for an image with range [vmin, vmax]"""
    coeff = -0.5 / (sigma_color * sigma_color)
    length = F32(float(vmax) - float(vmin))
    scale_index = F32(F32(EXP_BINS) / length)
    i = np.arange(EXP_BINS + 2, dtype=np.float32)
    val = (i / scale_index).astype(np.float64)
    return scale_index, np.exp(val * val * coeff).astype(np.float32)


def bilateral(img, minmax_mask=None):
    """cv2.bilateralFilter(img, 5, 0.5, 2.0) on float32 [H,W]: range weights interpolated from a 4096(+2)-bin
    table over [0, max - min] of the whole image (a copy when max - min < FLT_EPSILON), spatial weights
    exp(-r^2 / 8), reflect-101 borders.  Weights in float32 as cv2 computes them, sums in float64.
    Returns (filtered, (min, max))."""
    src = img if minmax_mask is None else img[minmax_mask]
    vmin, vmax = (float(src.min()), float(src.max())) if src.size else (0.0, 0.0)
    if abs(vmin - vmax) < FLT_EPSILON:
        return img.copy(), (vmin, vmax)
    scale_index, lut = bilateral_lut(vmin, vmax)
    h, w = img.shape
    p = np.pad(img, 2, mode="reflect")
    s = np.zeros((h, w), np.float64)
    ws = np.zeros((h, w), np.float64)
    for dy, dx, sw in space_taps():
        val = p[2 + dy:2 + dy + h, 2 + dx:2 + dx + w]
        alpha = np.abs(val - img) * scale_index
        if minmax_mask is not None:  # the mutant's range misses pixels outside the mask
            alpha = np.minimum(alpha, F32(EXP_BINS))
        idx = np.floor(alpha).astype(np.int64)
        alpha = alpha - idx.astype(np.float32)
        lo, hi = lut[idx], lut[idx + 1]
        wt = sw * (lo + alpha * (hi - lo))
        s += val.astype(np.float64) * wt
        ws += wt
    return (s / ws).astype(np.float32), (vmin, vmax)


def fill_stages(depth, cam_scale, scale_2_80m=1.0, mutant=None):
    """One frame: depth [H,W] (raw units, taken as float32), cam_scale, scale_2_80m -> dict of float32 [H,W]
    stages s1 .. s4, s5, s7_pre (after the fill iterations and the masked median: the bilateral's input),
    s7 (after the masked bilateral), s8 (inverted), out ([H,W] rescaled), int top1 / top2 [W], V [H,W] bool and
    minmax (the bilateral's (min, max))."""
    if mutant is not None and mutant not in MUTANTS:
        raise ValueError(f"unknown mutant {mutant!r}")
    cs, s2s = F32(cam_scale), F32(scale_2_80m)
    d = (np.asarray(depth, np.float32) / cs) * s2s
    h = d.shape[0]
    border = 0.0 if mutant == "dilate_zero" else -np.inf
    mmode = "reflect" if mutant == "median_reflect" else "edge"
    near = (d > T) & (d <= F32(1.0))
    med = (d > F32(1.0)) & (d <= F32(2.0))
    far = d > F32(2.0)
    s1 = np.where(d > T, MAX_DEPTH - d, d)
    df = dilate(s1 * far, CROSS_3, border)
    dm = dilate(s1 * med, CROSS_5, border)
    dn = dilate(s1 * near, CROSS_7, border)
    s2 = s1.copy()
    for dil in (df, dm, dn):
        s2 = np.where(dil > T, dil, s2)
    s3 = erode(dilate(s2, FULL_5, border), FULL_5)
    s4 = np.where(s3 > T, median5(s3, mmode), s3)
    top1 = top_rows(s4)
    s5 = np.where(~(s4 > T) & _under(top1, h), dilate(s4, FULL_9, border), s4)
    top2 = top_rows(s5)
    under = _under(top1 if mutant == "top1_loop" else top2, h)
    s = s5.copy()
    for _ in range(5 if mutant == "five_iters" else 6):
        empty = ((s <= T) if mutant == "loop_le" else (s < T)) & under
        s = np.where(empty, dilate(s, FULL_5, border), s)
    V = (s > T) & under
    s7_pre = np.where(V, median5(s, mmode), s)
    if mutant == "v_after_median":
        V = (s7_pre > T) & under
    bl, minmax = bilateral(s7_pre, V if mutant == "minmax_valid" else None)
    s7 = np.where(V, bl, s7_pre)
    s8 = np.where(s7 > T, MAX_DEPTH - s7, s7)
    out = (s8 / s2s) * cs
    return dict(s1=s1, s2=s2, s3=s3, s4=s4, s5=s5, s7_pre=s7_pre, s7=s7, s8=s8, out=out, top1=top1, top2=top2,
                V=V, minmax=minmax)


def fill_missing(depth, cam_scale, scale_2_80m=1.0, mutant=None):
    """Basic_Utils.fill_missing(depth, cam_scale, scale_2_80m) as this module computes it: [H,W] float32"""
    return fill_stages(depth, cam_scale, scale_2_80m, mutant)["out"]


def bilateral_bound(minmax):
    """the kernel's bound on |bilateral - this module's bilateral| for a frame whose pre-bilateral image spans
    minmax = (min, max): 3 * 2^-20 * max(|min|, |max|)  (include/pvn3d_b200.h derives it)"""
    return 3.0 * 2.0 ** -20 * max(abs(minmax[0]), abs(minmax[1]))


def out_bound(minmax, cam_scale, scale_2_80m, ref_out=0.0):
    """the bound carried through step 11: the inversion's rounding (at most 2^-23 on either side), then the
    rescale's two roundings relative to the output"""
    return (bilateral_bound(minmax) + 2.0 ** -22) * float(cam_scale) / float(scale_2_80m) + \
        2.0 ** -21 * np.abs(ref_out)


def mutant_rejected(mutant_stages, s4, s5, s7, minmax):
    """True when a mutant's stages are told apart from (s4, s5, s7): s4 or s5 not bit-equal, or s7 farther
    than the bilateral bound anywhere"""
    if not (np.array_equal(mutant_stages["s4"], s4) and np.array_equal(mutant_stages["s5"], s5)):
        return True
    d = np.abs(mutant_stages["s7"].astype(np.float64) - np.asarray(s7, np.float64)).max()
    return bool(d > bilateral_bound(minmax))
