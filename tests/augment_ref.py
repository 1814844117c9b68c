"""numpy restatement of get_item's training augmentation (ycb_dataset.py / linemod_dataset.py of the reference),
each operation in the precision of the library the reference calls, given an explicit parameter record:

  ColorJitter(0.2, 0.2, 0.2, 0.05)   PIL 12.2 / torchvision 0.26: Image.blend in float32 with a truncating store
                                     (brightness against 0, contrast against the rounded mean of convert("L"),
                                     saturation against convert("L")), hue through PIL's RGB<->HSV with
                                     np.int32(h * 255).astype(np.uint8) added modulo 256
  rgb_add_noise                      cv2 4.13: BGR2HSV 8U (12-bit fixed-point tables), S/V scaled in float64 and
                                     truncated into uint16, HSV2BGR 8U (float32), filter2D with the float sharpen
                                     and motion kernels (float32 taps and sums), GaussianBlur 8U (the bit-exact
                                     fixed-point path, BORDER_REFLECT_101); YCB's noise in float32 from a given
                                     standard-normal field
  add_real_back                      the uint8 / float32 composite of colour and depth

tests/golden/make_golden_augment.py checks every function here against cv2 / PIL / torchvision and the reference's
own methods; tests/test_augment_gpu.py checks csrc/augment.cu against these functions.
"""
from __future__ import annotations

import math

import numpy as np

YCB, LINEMOD = "ycb", "linemod"
# frame kinds (include/pvn3d_b200.h): YCB real / syn, LineMOD real png / render / fuse
KIND_REAL, KIND_SYN = 0, 1
KIND_RENDER, KIND_FUSE = 1, 2

# ---- the parameter record (pvn3d_augment_params_t) -------------------------------------------------------------
from pvn3d_b200.augment import PASS_DTYPE, RECORD_DTYPE as PARAMS_DTYPE  # noqa: E402,F401

#: deliberately wrong variants (select with `with mutant(name):`), for tests that show the goldens tell them apart
MUTANTS = ("hsv2bgr_round", "sv_round", "blend_round", "contrast_floor", "gauss_plain", "reflect", "hue_clip",
           "back_rgb_order", "depth_keep_zero", "noise_round")
MUTANT = None


class mutant:
    def __init__(self, name):
        if name not in MUTANTS:
            raise ValueError(f"unknown mutant {name!r}")
        self.name = name

    def __enter__(self):
        global MUTANT
        MUTANT = self.name

    def __exit__(self, *exc):
        global MUTANT
        MUTANT = None


S_RANGE = {YCB: (1.25, 1.45), LINEMOD: (0.75, 1.25)}
V_RANGE = {YCB: (1.15, 1.35), LINEMOD: (0.85, 1.15)}


def blank_params(n: int) -> np.ndarray:
    """n records that change nothing: no jitter, no noise pass, no background"""
    p = np.zeros(n, PARAMS_DTYPE)
    p["order"] = np.arange(4)
    p["brightness"] = p["contrast"] = p["saturation"] = 1.0
    p["passes"]["s_factor"] = p["passes"]["v_factor"] = 1.0
    p["passes"]["ksize"] = 3
    return p


def host_draw(rng: np.random.Generator, dataset: str, kinds) -> np.ndarray:
    """Records drawn on the host with the reference's decision structure and distributions (not its streams)."""
    kinds = np.asarray(kinds)
    p = blank_params(len(kinds))
    for i, k in enumerate(kinds):
        r = p[i]
        r["kind"] = k
        r["jitter"] = 1 if dataset == YCB else int(k == KIND_REAL)
        if r["jitter"]:
            r["order"] = rng.permutation(4)
            r["brightness"], r["contrast"], r["saturation"] = rng.uniform(0.8, 1.2, 3).astype(np.float32)
            r["hue"] = np.float32(rng.uniform(-0.05, 0.05))
        noisy = k == (KIND_SYN if dataset == YCB else KIND_RENDER)
        if noisy:
            r["back"] = 1
            r["n_pass"] = 1 + int(rng.random() > 0.8)
            for q in range(r["n_pass"]):
                ps = r["passes"][q]
                ps["s_factor"] = rng.uniform(*S_RANGE[dataset])
                ps["v_factor"] = rng.uniform(*V_RANGE[dataset])
                if dataset == YCB:
                    ps["sharpen"] = int(rng.random() > 0.8)
                    ps["sharpen_w"] = rng.random() * 3 + 9
                ps["motion"] = int(rng.random() > 0.8)
                ps["angle"] = int(rng.random() * 360)
                ps["length"] = int(rng.random() * 15) + 1
                ps["gauss"] = int(rng.random() > 0.8)
                ps["ksize"] = 3 if rng.random() > 0.2 else 5
                ps["sigma"] = rng.random()
                if dataset == YCB:
                    ps["noise_sigma"] = rng.integers(15) if rng.random() > 0.2 else rng.integers(25)
                    ps["extra"] = int(rng.random() > 0.8)
                ps["noise_key"], ps["extra_key"] = rng.integers(0, 2**63, 2)
    return p


# ---- PIL 12.2 --------------------------------------------------------------------------------------------------
def pil_l(rgb: np.ndarray) -> np.ndarray:
    """Image.convert("L") of RGB: ITU-R 601-2 in 16-bit fixed point, rounded"""
    x = rgb.astype(np.int64)
    return ((x[..., 0] * 19595 + x[..., 1] * 38470 + x[..., 2] * 7471 + 0x8000) >> 16).astype(np.uint8)


def pil_blend(im1, im2, alpha) -> np.ndarray:
    """Image.blend(im1, im2, alpha): float32 in1 + alpha * (in2 - in1); truncating store, clamped outside [0, 1]"""
    a = np.float32(alpha)
    i1 = np.asarray(im1).astype(np.float32)
    t = i1 + a * (np.asarray(im2).astype(np.float32) - i1)
    if MUTANT == "blend_round":
        return np.clip(np.rint(t), 0, 255).astype(np.uint8)
    if 0.0 <= a <= 1.0:
        return t.astype(np.int64).astype(np.uint8)   # (UINT8) of a value in [0, 255]
    return np.where(t <= 0, 0, np.where(t >= 255, 255, np.trunc(np.clip(t, 0, 255)))).astype(np.uint8)


def pil_rgb2hsv(rgb: np.ndarray) -> np.ndarray:
    """Image.convert("HSV") of RGB (Convert.c rgb2hsv_row): float32 / float64 exactly as the C mixes them"""
    r, g, b = (rgb[..., i].astype(np.int64) for i in range(3))
    mx = np.maximum(r, np.maximum(g, b))
    mn = np.minimum(r, np.minimum(g, b))
    cr = (mx - mn).astype(np.float32)
    crs = np.where(cr == 0, np.float32(1), cr)
    with np.errstate(divide="ignore", invalid="ignore"):
        s = cr / np.where(mx == 0, 1, mx).astype(np.float32)
        rc = (mx - r).astype(np.float32) / crs
        gc = (mx - g).astype(np.float32) / crs
        bc = (mx - b).astype(np.float32) / crs
    h = np.where(r == mx, (bc - gc).astype(np.float32),
                 np.where(g == mx, (2.0 + rc.astype(np.float64) - bc).astype(np.float32),
                          (4.0 + gc.astype(np.float64) - rc).astype(np.float32)))
    h = np.fmod(h.astype(np.float64) / 6.0 + 1.0, 1.0).astype(np.float32)
    uh = np.clip((h.astype(np.float64) * 255.0).astype(np.int64), 0, 255)
    us = np.clip((s.astype(np.float64) * 255.0).astype(np.int64), 0, 255)
    same = mn == mx
    out = np.stack([np.where(same, 0, uh), np.where(same, 0, us), mx], -1)
    return out.astype(np.uint8)


def _c_round(x):
    return np.where(x >= 0, np.floor(x + 0.5), np.ceil(x - 0.5))


def pil_hsv2rgb(hsv: np.ndarray) -> np.ndarray:
    """Image.convert("RGB") of HSV (Convert.c hsv2rgb)"""
    h, s, v = (hsv[..., i].astype(np.int64) for i in range(3))
    hf = h.astype(np.float32).astype(np.float64)
    i = np.floor(hf * 6.0 / 255.0).astype(np.int64)
    f = (hf * 6.0 / 255.0 - i.astype(np.float32)).astype(np.float32).astype(np.float64)
    fs = (s.astype(np.float32).astype(np.float64) / 255.0).astype(np.float32).astype(np.float64)
    vf = v.astype(np.float64)
    p = np.clip(_c_round(vf * (1.0 - fs)), 0, 255).astype(np.int64)
    q = np.clip(_c_round(vf * (1.0 - (fs.astype(np.float32) * f.astype(np.float32)).astype(np.float64))), 0,
                255).astype(np.int64)   # fs * f is a float32 product in the C
    t = np.clip(_c_round(vf * (1.0 - fs * (1.0 - f))), 0, 255).astype(np.int64)
    sec = i % 6
    r = np.choose(sec, [v, q, p, p, t, v])
    g = np.choose(sec, [t, v, v, q, p, p])
    b = np.choose(sec, [p, p, t, v, v, q])
    out = np.stack([r, g, b], -1)
    out = np.where((s == 0)[..., None], v[..., None], out)
    return out.astype(np.uint8)


def hue_shift(hue: float) -> int:
    """torchvision's np.int32(hue_factor * 255).astype(np.uint8), hue_factor a float32 widened to float"""
    return int(np.int32(float(np.float32(hue)) * 255) & 0xFF)


def jitter_op(img: np.ndarray, op: int, p) -> np.ndarray:
    """one ColorJitter step on an RGB uint8 [H,W,3] image: 0 brightness, 1 contrast, 2 saturation, 3 hue"""
    if op == 0:
        return pil_blend(np.zeros_like(img), img, p["brightness"])
    if op == 1:
        mean = int(float(pil_l(img).astype(np.int64).sum()) / (img.shape[0] * img.shape[1])
                   + (0.0 if MUTANT == "contrast_floor" else 0.5))
        return pil_blend(np.full_like(img, mean), img, p["contrast"])
    if op == 2:
        return pil_blend(np.repeat(pil_l(img)[..., None], 3, -1), img, p["saturation"])
    hsv = pil_rgb2hsv(img)
    if MUTANT == "hue_clip":
        hsv[..., 0] = np.clip(hsv[..., 0].astype(np.int64) + np.int32(float(np.float32(p["hue"])) * 255), 0, 255)
    else:
        hsv[..., 0] = (hsv[..., 0].astype(np.int64) + hue_shift(p["hue"])) & 0xFF
    return pil_hsv2rgb(hsv)


def color_jitter(img: np.ndarray, p) -> np.ndarray:
    for op in p["order"]:
        img = jitter_op(img, int(op), p)
    return img


# ---- cv2 4.13 --------------------------------------------------------------------------------------------------
_HSV_SHIFT = 12


def _tables():
    i = np.arange(256, dtype=np.float64)
    with np.errstate(divide="ignore"):
        sdiv = np.where(i == 0, 0, np.rint((255 << _HSV_SHIFT) / i)).astype(np.int64)
        hdiv = np.where(i == 0, 0, np.rint((180 << _HSV_SHIFT) / (6.0 * i))).astype(np.int64)
    return sdiv, hdiv


SDIV, HDIV = _tables()


def cv_bgr2hsv(img: np.ndarray) -> np.ndarray:
    """cv2.cvtColor(img, COLOR_BGR2HSV) for uint8: H in [0, 180)"""
    b, g, r = (img[..., i].astype(np.int64) for i in range(3))
    v = np.maximum(b, np.maximum(g, r))
    diff = v - np.minimum(b, np.minimum(g, r))
    half = 1 << (_HSV_SHIFT - 1)
    s = (diff * SDIV[v] + half) >> _HSV_SHIFT
    h = np.where(v == r, g - b, np.where(v == g, b - r + 2 * diff, r - g + 4 * diff))
    h = (h * HDIV[diff] + half) >> _HSV_SHIFT
    h = np.where(h < 0, h + 180, h)
    return np.stack([h, s, v], -1).astype(np.uint8)


_SECTOR = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]])


def _fma32(a, b, c):
    """float32 fused multiply-add (the product of two float32 is exact in float64)"""
    return (a.astype(np.float64) * b.astype(np.float64) + c).astype(np.float32)


#: cv2 4.13 converts each row in vectors of 32 pixels (its AVX2 dispatch) and the last width % 32 pixels one by one
CV_VECTOR = 32


def cv_hsv2bgr(hsv: np.ndarray, vector: bool = True) -> np.ndarray:
    """cv2.cvtColor(hsv, COLOR_HSV2BGR) for uint8 as cv2 4.13 computes it: float32, s and v scaled by 1/255,
    1 - s*h and 1 - s*(1-h) each one fused multiply-add, the result times 255 -- truncated in the vector loop,
    rounded to nearest even in the per-pixel tail of a row (vector=False)"""
    f32 = np.float32
    h = hsv[..., 0].astype(f32) * f32(6.0 / 180)
    s = hsv[..., 1].astype(f32) * f32(1 / 255)
    v = hsv[..., 2].astype(f32) * f32(1 / 255)
    sec = np.floor(h).astype(np.int64)
    h = h - sec.astype(f32)
    sec %= 6
    one = f32(1)
    tab = np.stack([v, v * (one - s), v * _fma32(-s, h, one), v * _fma32(-s, one - h, one)], -1)
    out = np.take_along_axis(tab, _SECTOR[sec], -1)
    out = np.where((s == 0)[..., None], v[..., None], out)
    rnd = np.rint if (MUTANT == "hsv2bgr_round" or not vector) else np.trunc
    return np.clip(rnd(out * f32(255)), 0, 255).astype(np.uint8)


def hsv_scale(img: np.ndarray, s_factor: float, v_factor: float) -> np.ndarray:
    """rgb_add_noise's HSV augmentor: BGR2HSV, S and V times float64 factors truncated into uint16 and clipped,
    HSV2BGR (YCB feeds it an RGB image; the conversion treats its first channel as blue all the same)"""
    hsv = cv_bgr2hsv(img).astype(np.uint16)
    if MUTANT == "sv_round":
        hsv[:, :, 1] = np.rint(hsv[:, :, 1] * float(s_factor))
        hsv[:, :, 2] = np.rint(hsv[:, :, 2] * float(v_factor))
    else:
        hsv[:, :, 1] = hsv[:, :, 1] * float(s_factor)
        hsv[:, :, 2] = hsv[:, :, 2] * float(v_factor)
    hsv[:, :, 1] = np.clip(hsv[:, :, 1], 0, 255)
    hsv[:, :, 2] = np.clip(hsv[:, :, 2], 0, 255)
    hsv = hsv.astype(np.uint8)
    split = hsv.shape[1] // CV_VECTOR * CV_VECTOR
    return np.concatenate([cv_hsv2bgr(hsv[:, :split]), cv_hsv2bgr(hsv[:, split:], vector=False)], 1)


def reflect101(i, n):
    """BORDER_REFLECT_101 index"""
    if n == 1:
        return np.zeros_like(i)
    if MUTANT == "reflect":                     # BORDER_REFLECT: the edge pixel repeated
        period = 2 * n
        i = np.where(i < 0, -i - 1, i) % period
        return np.where(i >= n, period - 1 - i, i)
    period = 2 * (n - 1)
    i = np.abs(i) % period
    return np.where(i >= n, period - i, i)


# GaussianBlur 8U ---------------------------------------------------------------------------------------------
_SMALL_GAUSS = {3: [0.25, 0.5, 0.25], 5: [0.0625, 0.25, 0.375, 0.25, 0.0625]}


def gaussian_kernel_f64(ksize: int, sigma: float) -> list[float]:
    """getGaussianKernelBitExact: the small fixed tables for sigma <= 0, else exp(-x^2 / (8 sigma^2)) over
    x = 1-n, 3-n, ... in float64 (IEEE; cv's softdouble is IEEE float64 too), normalised by the sum"""
    if sigma <= 0:
        return list(_SMALL_GAUSS[ksize])
    s = float(sigma)
    s2 = s * s
    scale2 = -0.125 / s2 if s2 > 0 else -math.inf     # IEEE: a sigma whose square underflows leaves the centre tap
    half = (ksize - 1) // 2
    vals, tot = [], 0.0
    x = 1 - ksize
    for _ in range(half):
        t = math.exp(float(x * x) * scale2)
        vals.append(t)
        tot += t
        x += 2
    tot = tot * 2.0 + 1.0
    inv = 1.0 / tot
    side = [v * inv for v in vals]
    return side + [inv] + side[::-1]


def gaussian_kernel_fixed(ksize: int, sigma: float) -> np.ndarray:
    """getGaussianKernelFixedPoint_ED with 8 fractional bits: error-diffused rounding of the outer taps, the
    centre takes what is left of 256"""
    k = gaussian_kernel_f64(ksize, sigma)
    half = ksize // 2
    out = np.zeros(ksize, np.int64)
    err, tot = 0.0, 0
    for i in range(half):
        adj = k[i] * 256.0 + err
        v = int(np.rint(adj))
        err = 0.0 if MUTANT == "gauss_plain" else adj - v
        out[i] = out[ksize - 1 - i] = v
        tot += v
    out[half] = 256 - 2 * tot
    return out


def gaussian_blur(img: np.ndarray, ksize: int, sigma: float) -> np.ndarray:
    """cv2.GaussianBlur(img, (k, k), sigma) on uint8 [H,W,C]: rows then columns in fixed point, BORDER_REFLECT_101,
    out = (sum_y ky * (sum_x kx * x) + 2^15) >> 16"""
    k = gaussian_kernel_fixed(ksize, sigma)
    hgt, wid = img.shape[:2]
    r = ksize // 2
    x = img.astype(np.int64)
    xs = reflect101(np.arange(-r, wid + r), wid)
    ys = reflect101(np.arange(-r, hgt + r), hgt)
    xp = x[:, xs]
    row = sum(k[i] * xp[:, i:i + wid] for i in range(ksize))
    rp = row[ys]
    col = sum(k[i] * rp[i:i + hgt] for i in range(ksize))
    return np.minimum((col + (1 << 15)) >> 16, 255).astype(np.uint8)


# filter2D with a float kernel ----------------------------------------------------------------------------------
def motion_line(angle: int, length: int):
    """linear_motion_blur's kernel before normalisation: the kernel size a and the taps (row, col) cv2.line sets
    in an a x a grid from (a//2, a//2) to (int(cos*len + a//2), int(sin*len + a//2)); 8-connected, clipped to the
    grid as cv::clipLine does.  a == 0 means the image is returned unchanged."""
    rad = np.deg2rad(angle)
    dx, dy = np.cos(rad), np.sin(rad)
    a = int(max(abs(dx), abs(dy)) * length * 2)
    if a <= 0:
        return 0, []
    c = a // 2
    x1, y1 = c, c
    x2, y2 = int(dx * length + c), int(dy * length + c)
    # cv::clipLine (pt1 is always inside)
    right = bottom = a - 1
    c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8
    if c2:
        if c2 & 12:
            t = 0 if c2 < 8 else bottom
            x2 += int(float(t - y2) * (x2 - x1) / (y2 - y1))
            y2 = t
            c2 = (x2 < 0) + (x2 > right) * 2
        if c2:
            t = 0 if c2 == 1 else right
            y2 += int(float(t - x2) * (y2 - y1) / (x2 - x1))
            x2 = t
    return a, bresenham8(x1, y1, x2, y2)


def bresenham8(x1, y1, x2, y2):
    """cv::LineIterator, 8-connected, left to right: the pixels (row, col) of the segment"""
    if x2 < x1:
        x1, y1, x2, y2 = x2, y2, x1, y1
    dx, dy = x2 - x1, y2 - y1
    sx, sy = 1, 1
    if dy < 0:
        dy, sy = -dy, -1
    vert = dy > dx
    if vert:
        dx, dy = dy, dx
    err = dx - (dy + dy)
    plus, minus = dx + dx, -(dy + dy)
    x, y = x1, y1
    pts = []
    for _ in range(dx + 1):
        pts.append((y, x))
        mask = err < 0
        err += minus + (plus if mask else 0)
        if vert:
            y += sy
            x += sx if mask else 0
        else:
            x += sx
            y += sy if mask else 0
    return pts


def motion_kernel(angle: int, length: int) -> np.ndarray | None:
    """the normalised float64 a x a motion kernel, None when linear_motion_blur returns the image unchanged"""
    a, pts = motion_line(angle, length)
    if a == 0:
        return None
    k = np.zeros((a, a))
    for (y, x) in pts:
        k[y, x] = 1.0
    s = k.sum()
    if s == 0:
        k[a // 2, a // 2] = 1.0
    else:
        k /= s
    return k


def sharpen_kernel(w: float) -> np.ndarray:
    k = -np.ones((3, 3))
    k[1, 1] = w
    return k / k.sum()


def filter2d(img: np.ndarray, kern: np.ndarray) -> np.ndarray:
    """cv2.filter2D(img, -1, kern) as a direct correlation: float32 taps, anchor (a//2, a//2), BORDER_REFLECT_101,
    float32 sums over the nonzero taps in row-major order, rounded to nearest even and saturated.  cv2 may sum in
    another order, or through a DFT for large kernels: it is within 1 of this."""
    kh, kw = kern.shape
    hgt, wid = img.shape[:2]
    k32 = kern.astype(np.float32)
    x = img.astype(np.float32)
    acc = np.zeros(img.shape, np.float32)
    for ky in range(kh):
        ys = reflect101(np.arange(hgt) + ky - kh // 2, hgt)
        for kx in range(kw):
            if k32[ky, kx] == 0:
                continue
            xs = reflect101(np.arange(wid) + kx - kw // 2, wid)
            acc = acc + k32[ky, kx] * x[ys][:, xs]
    return np.clip(np.rint(acc), 0, 255).astype(np.uint8)


# noise and the composite ---------------------------------------------------------------------------------------
def add_noise(img: np.ndarray, field: np.ndarray, sigma) -> np.ndarray:
    """gaussian_noise / the extra noise with a given standard-normal field, in float32: clip(x + n * sigma), then
    the uint8 truncation"""
    t = img.astype(np.float32) + field.astype(np.float32) * np.float32(sigma)
    if MUTANT == "noise_round":
        t = np.rint(t)
    return np.clip(t, np.float32(0), np.float32(255)).astype(np.uint8)


def add_real_back(rgb, labels, dpt, back_rgb, back_labels, back_dpt, dataset):
    """add_real_back given the background frame: rgb uint8 [H,W,3] in the network's channel order, labels [H,W],
    dpt float32 [H,W] (depth before the composite), back_rgb [H,W,3] RGB as decoded, back_labels [H,W] or [H,W,3],
    back_dpt [H,W].  Returns (rgb, dpt)."""
    bk = (back_labels <= 0).astype(np.uint8)
    if bk.ndim == 2:
        bk3 = np.repeat(bk[:, :, None], 3, 2)
    else:
        bk3, bk = bk, bk[:, :, 0]
    back = back_rgb[:, :, :3] * bk3
    if dataset == LINEMOD and MUTANT != "back_rgb_order":
        back = back[:, :, ::-1]
    dpt_back = back_dpt.astype(np.float32) * bk.astype(np.float32)
    msk = np.repeat((labels <= 0).astype(np.uint8)[:, :, None], 3, 2)
    rgb = rgb * (msk == 0).astype(np.uint8) + back * msk
    keep = dpt.astype(np.float64) > 1e-6
    if MUTANT == "depth_keep_zero":
        keep = np.ones_like(keep)
    dpt = np.where(keep, dpt.astype(np.float32), dpt_back).astype(np.float32)
    return rgb, dpt


# one noise pass and the whole stage ---------------------------------------------------------------------------
def noise_pass(img, ps, dataset, noise=None, extra=None, stages=None):
    """rgb_add_noise with the record's pass `ps`; noise / extra are the standard-normal fields [H,W,3]"""
    img = hsv_scale(img, ps["s_factor"], ps["v_factor"])
    st = [img]
    if dataset == YCB and ps["sharpen"]:
        img = filter2d(img, sharpen_kernel(ps["sharpen_w"]))
    st.append(img)
    if ps["motion"]:
        k = motion_kernel(int(ps["angle"]), int(ps["length"]))
        if k is not None:
            img = filter2d(img, k)
    st.append(img)
    if ps["gauss"]:
        img = gaussian_blur(img, int(ps["ksize"]), float(ps["sigma"]))
    st.append(img)
    if dataset == YCB:
        img = add_noise(img, noise, int(ps["noise_sigma"]))
        if ps["extra"]:
            img = add_noise(img, extra, 7.0)
    st.append(img)
    if stages is not None:
        stages.extend(st)
    return img


def augment_frame(rgb, dpt, labels, back_rgb, back_labels, back_dpt, p, dataset, noise=None):
    """get_item's augmentation of one frame from its record.  rgb [H,W,3] uint8 RGB as decoded, dpt [H,W] float32,
    labels [H,W] uint8; noise [2 passes, 2 (noise, extra), H, W, 3] float32 standard normals.  Returns
    (rgb [3,H,W] in the network's channel order, dpt, stages) with stages the images after the jitter (and the
    flip), each step of pass 1, the composite and each step of pass 2 (unused passes repeat the last image)."""
    img = color_jitter(rgb, p) if p["jitter"] else rgb.copy()
    if dataset == LINEMOD:
        img = img[:, :, ::-1].copy()
    stages = [img]
    dpt = dpt.astype(np.float32)
    for q in range(2):
        if q < p["n_pass"]:
            img = noise_pass(img, p["passes"][q], dataset, None if noise is None else noise[q, 0],
                             None if noise is None else noise[q, 1], stages)
        else:
            stages.extend([img] * 5)
        if q == 0:
            if p["back"]:
                img, dpt = add_real_back(img, labels, dpt, back_rgb, back_labels, back_dpt, dataset)
            stages.append(img)
    return np.ascontiguousarray(img.transpose(2, 0, 1)), dpt, stages


N_STAGES = 12
