"""NumPy statement of the full-resolution scene of eval_icp's refinement (pvn3d/eval_icp.py:224-291,
388-422) as pvn3d_b200's DepthIcpRefiner runs it -- a checker, written from the documented steps:

1. back-projection (Basic_Utils.dpt_2_cld, lib/utils/basic_utils.py:381-399) of every pixel in raster
   order, float32: valid = dpt > 1e-6; pt2 = dpt / cam_scale; pt0 = ((col - cx) * pt2) / fx;
   pt1 = ((row - cy) * pt2) / fy; invalid pixels (0, 0, 0).
2. label fill (fill_label_item): every valid pixel takes the label of its nearest sampled point by the
   float64 squared distance (dx*dx + dy*dy) + dz*dz, lowest index on exact ties; invalid pixels 0.
3. per object: its pixels in raster order, the strided selection of max_pts, skipped below min_pts,
   the biggest flat mean-shift cluster, then my_icp.
"""
from __future__ import annotations

import numpy as np

from oracle import flat_meanshift_oracle, icp_oracle


def dpt_2_cld(dpt: np.ndarray, cam_scale, K) -> tuple:
    """step 1 for one [H,W] frame -> (cloud [H*W,3] f32, valid [H*W] bool)"""
    d = np.asarray(dpt, np.float32)
    h, w = d.shape
    k = np.asarray(K, np.float32)
    cs = np.float32(cam_scale)
    rows = np.repeat(np.arange(h, dtype=np.float32), w)
    cols = np.tile(np.arange(w, dtype=np.float32), h)
    d = d.reshape(-1)
    valid = d > np.float32(1e-6)
    pt2 = d / cs
    pt0 = ((cols - k[0, 2]) * pt2) / k[0, 0]
    pt1 = ((rows - k[1, 2]) * pt2) / k[1, 1]
    cloud = np.stack([pt0, pt1, pt2], 1).astype(np.float32)
    cloud[~valid] = 0.0
    return cloud, valid


def sqdist64(q: np.ndarray, p: np.ndarray) -> np.ndarray:
    """[Q,P] float64 squared distances, (dx*dx + dy*dy) + dz*dz"""
    d = q[:, None, :].astype(np.float64) - p[None, :, :].astype(np.float64)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def fill_label(cloud: np.ndarray, valid: np.ndarray, pcld: np.ndarray, point_labels: np.ndarray,
               chunk: int = 512) -> tuple:
    """step 2 for one frame by brute force -> (labels [P] i32, nn index [P] i64, -1 where invalid)"""
    idx = np.full(len(cloud), -1, np.int64)
    q_at = np.nonzero(valid)[0]
    for s in range(0, len(q_at), chunk):
        sel = q_at[s:s + chunk]
        idx[sel] = np.argmin(sqdist64(cloud[sel], pcld), axis=1)    # first minimum: lowest index
    labels = np.where(idx >= 0, np.asarray(point_labels)[np.maximum(idx, 0)], 0).astype(np.int32)
    return labels, idx


def object_fit(model, cloud: np.ndarray, labels: np.ndarray, cls: int, init, max_pts: int, min_pts: int,
               bw: float = 0.06, max_iter: int = 500, tol: float = 1e-9, cluster_max_iter: int = 300,
               nn=icp_oracle.nearest):
    """step 3 for one (frame, class): labels [H*W] with 0 on invalid pixels.  Returns None when the
    object is skipped (fewer than min_pts pixels), else (T 4x4, distances, i, kept pixel indices)."""
    if (np.asarray(labels) == cls).sum() < min_pts:
        return None
    sel = icp_oracle.select(labels, cls, max_pts)
    B = np.asarray(cloud)[sel]
    kept = flat_meanshift_oracle.biggest_cluster(B.astype(np.float64), bw, cluster_max_iter)
    T, d, i = icp_oracle.my_icp(model, B[kept], init, max_iter, tol, nn=nn)
    return T, d, i, sel[kept]
