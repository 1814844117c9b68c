"""NumPy float64 statement of my_icp (reference lib/utils/icp/icp.py:141-192) and of the scene-point
selection of pvn3d_b200's batched ICP -- a checker, written from the documented semantics.

my_icp: src = init * A (homogeneous); per iteration every scene point finds its nearest point of src
(brute force, lowest index on exact ties), T = best_fit_transform(src[idx], B), src = T src; stop when
|prev - mean(d)| < tol with prev starting at 0.  Returns (best_fit_transform(A, src), d, i).
"""
from __future__ import annotations

import numpy as np


def best_fit_transform(A: np.ndarray, B: np.ndarray) -> np.ndarray:
    """least-squares rigid A -> B (SVD with the reflection fix), 4x4 float64.  Float32 input keeps numpy's
    float32 arithmetic for its centroid and centred points (sequential float32 sum along axis 0)."""
    ca, cb = A.mean(axis=0), B.mean(axis=0)
    H = (A - ca).T @ (B - cb)
    U, _, Vt = np.linalg.svd(H)
    R = Vt.T @ U.T
    if np.linalg.det(R) < 0:
        Vt[2, :] *= -1
        R = Vt.T @ U.T
    T = np.identity(4)
    T[:3, :3] = R
    T[:3, 3] = cb - R @ ca
    return T


def nearest(queries: np.ndarray, pts: np.ndarray, chunk: int = 256):
    """exact float64 nearest point of pts for every query: (distances, indices), lowest index on ties
    (np.argmin keeps the first minimum)"""
    d_out = np.empty(len(queries))
    i_out = np.empty(len(queries), np.int64)
    for s in range(0, len(queries), chunk):
        q = queries[s:s + chunk]
        d2 = ((q[:, None, :] - pts[None, :, :]) ** 2).sum(-1)
        i = np.argmin(d2, axis=1)
        i_out[s:s + chunk] = i
        d_out[s:s + chunk] = np.sqrt(d2[np.arange(len(q)), i])
    return d_out, i_out


def my_icp(A, B, init_pose=None, max_iterations=20, tolerance=0.001, nn=nearest):
    """nn(queries, pts) -> (distances, indices): the brute force by default; a faster exact search
    may stand in for it on large batches"""
    A = np.asarray(A)  # kept as given: the final fit below takes A itself (float32 in eval_icp)
    B = np.asarray(B, np.float64)
    src = np.ones((4, len(A)))
    src[:3] = A.T
    if init_pose is not None:
        src = np.asarray(init_pose, np.float64) @ src
    prev = 0.0
    for i in range(max_iterations):
        distances, idx = nn(B, src[:3].T)
        T = best_fit_transform(src[:3, idx].T, B)
        src = T @ src
        mean = np.mean(distances)
        if np.abs(prev - mean) < tolerance:
            break
        prev = mean
    return best_fit_transform(A, src[:3].T), distances, i


def select(mask_row: np.ndarray, cls: int, max_pts: int) -> np.ndarray:
    """point indices of class `cls` in one frame's mask, as the batched refiner takes them: ascending
    index, and the points at positions floor(j * cnt / max_pts) when there are more than max_pts"""
    idx = np.nonzero(np.asarray(mask_row) == cls)[0]
    cnt = len(idx)
    if cnt > max_pts:
        idx = idx[(np.arange(max_pts, dtype=np.int64) * cnt) // max_pts]
    return idx
