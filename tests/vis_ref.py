"""A vectorised numpy restatement of demo.py's pose overlay (demo.py:122-145) and of the reference helpers it composes:
Basic_Utils.project_p3d (basic_utils.py:306-313), draw_p2ds (:315-323, one cv2.circle(img, c, r, color, -1) per point)
and get_label_color(mode=1) (:346-379).  Every operation is spelled out, so the order the GPU kernel must follow is
visible here:

  * the transform np.dot(mesh, R.T) + t and the projection np.dot(p3d * cam_scale, K.T) in float64, three products
    summed left to right, each product and sum rounded on its own (numpy's elementwise ops: no FMA);
  * z set to 1 where z < 1e-8 (NaN stays NaN), np.around (half to even), then numpy's x86-64 astype(np.int32): NaN and
    anything outside the int32 range become INT_MIN;
  * draw_p2ds's clip to [0, w] x [0, h] (not w - 1, h - 1), then the disc {dx^2 + dy^2 <= r^2} cut to the image;
  * cv2's colour conversion: each channel rounded half to even and saturated to [0, 255].

Shared by tests/golden/make_golden_vis.py (which checks it against the reference while recording) and the tests.
"""
import hashlib

import numpy as np

INT_MIN = np.int32(-2 ** 31)


def to_int32(v: np.ndarray) -> np.ndarray:
    """astype(np.int32) of an integral float64 array as numpy does it on x86-64"""
    ok = (v >= -2147483648.0) & (v <= 2147483647.0)
    out = np.full(v.shape, INT_MIN, np.int32)
    out[ok] = v[ok].astype(np.int32)
    return out


def dot3(q0, q1, q2, row):
    return (q0 * row[0] + q1 * row[1]) + q2 * row[2]


def transform(mesh: np.ndarray, pose: np.ndarray) -> np.ndarray:
    """[P,3] float64: np.dot(mesh, pose[:, :3].T) + pose[:, 3], the float32 mesh promoted"""
    m = np.asarray(mesh).astype(np.float64)
    pose = np.asarray(pose, np.float64)
    return np.stack([dot3(m[:, 0], m[:, 1], m[:, 2], pose[j, :3]) + pose[j, 3] for j in range(3)], 1)


def project_raw(p3d: np.ndarray, cam_scale: float, K: np.ndarray) -> np.ndarray:
    """[P,2] float64 before rounding: (u / d, v / d) of project_p3d"""
    q = p3d * cam_scale
    K = np.asarray(K, np.float64)
    u, v, d = (dot3(q[:, 0], q[:, 1], q[:, 2], K[j]) for j in range(3))
    with np.errstate(invalid="ignore"):
        d = np.where(d < 1e-8, 1.0, d)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        return np.stack([u / d, v / d], 1)


def project(p3d: np.ndarray, cam_scale: float, K: np.ndarray) -> np.ndarray:
    """Basic_Utils.project_p3d: [P,2] int32"""
    return to_int32(np.around(project_raw(p3d, cam_scale, K)))


def clip(p2ds: np.ndarray, h: int, w: int) -> np.ndarray:
    """draw_p2ds's clip (a copy): x to [0, w], y to [0, h]"""
    out = np.array(p2ds, copy=True)
    out[:, 0] = np.clip(out[:, 0], 0, w)
    out[:, 1] = np.clip(out[:, 1], 0, h)
    return out


def disc(r: int) -> np.ndarray:
    """[m,2] (dx, dy) with dx^2 + dy^2 <= r^2"""
    d = np.arange(-r, r + 1)
    dx, dy = np.meshgrid(d, d)
    keep = dx * dx + dy * dy <= r * r
    return np.stack([dx[keep], dy[keep]], 1)


def cv_color(color) -> np.ndarray:
    """[3] uint8 cv2 paints for `color` (1 to 4 numbers; missing channels 0; rint, then INT_MIN for NaN or outside
    int32 as cvRound gives on x86-64, then saturate)"""
    v = np.zeros(3, np.float64)
    c = np.asarray(color, np.float64).reshape(-1)[:3]
    v[:c.size] = c
    q = to_int32(np.rint(v)).astype(np.int64)
    return np.clip(q, 0, 255).astype(np.uint8)


def label_color(cls_id: int, n_obj: int = 22) -> tuple:
    """get_label_color(cls_id, n_obj, mode=1)"""
    m = 255 * 255 * 255 // n_obj * cls_id
    return (m // 255 // 255, (m // 255) % 255, m % 255)


def draw(img: np.ndarray, p2ds: np.ndarray, r: int, color) -> np.ndarray:
    """draw_p2ds on clipped points, vectorised: img [H,W,3] u8 painted in place and returned"""
    h, w = img.shape[:2]
    col = cv_color(color)
    if len(p2ds) == 0:
        return img
    for dx, dy in disc(int(r)):
        x = p2ds[:, 0].astype(np.int64) + dx
        y = p2ds[:, 1].astype(np.int64) + dy
        ok = (x >= 0) & (x < w) & (y >= 0) & (y < h)
        img[y[ok], x[ok]] = col
    return img


def overlay_frame(img, meshes, poses, present, order, K, colors, r=1, cam_scale=1.0):
    """demo.py's loop on one frame: for each class of `order` that is predicted (present), its mesh moved by its
    pose, projected, clipped and drawn in colors[class].  Returns (img, [clipped p2ds of each drawn slot])."""
    h, w = img.shape[:2]
    drawn = []
    for c in np.asarray(order).reshape(-1):
        c = int(c)
        if c < 1 or c >= len(present) or not present[c]:
            continue
        p2ds = clip(project(transform(meshes[c], poses[c]), cam_scale, K), h, w)
        draw(img, p2ds, r, colors[c])
        drawn.append(p2ds)
    return img, drawn


def background(seed: int, h: int, w: int) -> np.ndarray:
    """the seeded uint8 [H,W,3] frame a case draws on"""
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def sha(img: np.ndarray) -> bytes:
    return hashlib.sha256(np.ascontiguousarray(img).tobytes()).digest()


def changed(before: np.ndarray, after: np.ndarray):
    """(flat pixel indices int32, their values [m,3] u8) where after differs from before"""
    idx = np.nonzero((before != after).any(-1).reshape(-1))[0].astype(np.int32)
    return idx, after.reshape(-1, 3)[idx]


def rebuild(before: np.ndarray, idx: np.ndarray, vals: np.ndarray) -> np.ndarray:
    out = before.copy()
    out.reshape(-1, 3)[idx] = vals
    return out


def near_ties(raw: np.ndarray, tol: float = 1e-9) -> int:
    """how many finite projected coordinates lie within tol px of a .5 tie, where the summation order could matter"""
    f = raw[np.isfinite(raw)]
    return int(np.count_nonzero(np.abs(np.abs(f - np.floor(f)) - 0.5) <= tol))
