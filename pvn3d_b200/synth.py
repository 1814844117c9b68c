"""Synthetic RGB-D frames of the shapes BASELINE.json names (recipe pinned in SURVEY section 8d).

One frame = what the reference's data loader + network heads hand to the hot path:
    cld_rgb_nrm [N,9] f32  xyz | rgb(0..255) | normal            -> Pointnet2MSG     (hot path A)
    pcld [N,3], labels [N] i64, ctr_of [1,N,3], kp_of [K,N,3]    -> cal_frame_poses  (hot path B)
plus ground truth (RTs, class ids) for sanity checks.  Geometry: a background plane at z = 1.2 m
and one sphere per object instance, rendered into a 480x640 depth image and back-projected exactly
like Basic_Utils.dpt_2_cld (reference basic_utils.py:381-399); N pixels are kept in raster order as
the reference sampler does (ycb_dataset.py:227-231).  Votes are the true keypoints/centre of a
random pose plus N(0, 5 mm) noise, with 10 % of each instance's points voting uniformly at random
inside the cloud's bounding box.  Seeds: seed = 1000*config_id + frame_idx.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import numpy as np

from . import fixtures

H, W = 480, 640
K_LINEMOD = np.array([[572.4114, 0., 325.2611], [0., 573.57043, 242.04899], [0., 0., 1.]])   # common.py:138-140
K_YCB1 = np.array([[1066.778, 0., 312.9869], [0., 1067.487, 241.3109], [0., 0., 1.0]])       # common.py:144-146


@dataclass
class Frame:
    cld_rgb_nrm: np.ndarray   # [N,9] f32
    pcld: np.ndarray          # [N,3] f32
    labels: np.ndarray        # [N] i64
    ctr_of: np.ndarray        # [1,N,3] f32
    kp_of: np.ndarray         # [K,N,3] f32
    cls_ids: np.ndarray       # [n_inst] i64 (class id of each instance)
    RTs: np.ndarray           # [n_inst,3,4] f64 ground-truth poses
    obj_id: Optional[int] = None   # LineMOD object id whose fixtures were used


def _haar_rotation(rng) -> np.ndarray:
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _render(K, centres, radii, rng):
    """depth image [H,W] f32 and instance-index image (0 = plane, i+1 = sphere i)"""
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    v, u = np.mgrid[0:H, 0:W]
    dx, dy = (u - cx) / fx, (v - cy) / fy
    dn2 = dx * dx + dy * dy + 1.0
    depth = (1.2 + rng.normal(0.0, 0.002, size=(H, W)))
    inst = np.zeros((H, W), np.int32)
    for i, (c, r) in enumerate(zip(centres, radii)):
        bq = dx * c[0] + dy * c[1] + c[2]          # d . c
        disc = bq * bq - dn2 * (c @ c - r * r)
        hit = disc > 0
        t = (bq - np.sqrt(np.where(hit, disc, 0.0))) / dn2   # nearest intersection; z == t since d_z = 1
        closer = hit & (t < depth)
        depth = np.where(closer, t, depth)
        inst = np.where(closer, i + 1, inst)
    return depth.astype(np.float32), inst


def _back_project(depth, K):
    """Basic_Utils.dpt_2_cld with cam_scale = 1: returns cld [H*W,3] f32 (all pixels are valid)."""
    dpt = depth.flatten()[:, None].astype(np.float32)
    cols = np.tile(np.arange(W, dtype=np.float32), H)[:, None]
    rows = np.repeat(np.arange(H, dtype=np.float32), W)[:, None]
    pt0 = (cols - np.float32(K[0][2])) * dpt / np.float32(K[0][0])
    pt1 = (rows - np.float32(K[1][2])) * dpt / np.float32(K[1][1])
    return np.concatenate((pt0, pt1, dpt), axis=1).astype(np.float32)


def make_frame(shape: str = "linemod", n_points: int = fixtures.N_SAMPLE_POINTS, seed: int = 0,
               n_instances: Optional[int] = None, obj_frac: Optional[float] = None,
               outlier_frac: float = 0.10, vote_sigma: float = 0.005, lm_obj_id: Optional[int] = None) -> Frame:
    """shape: 'linemod' (1 instance, class id 1, ~25 % of the points) or 'ycb' (5 instances of distinct
    classes, ~8-11 % each; `n_instances` up to 6 per 3x2 image grid, or up to 12 on a 4x3 grid)."""
    rng = np.random.default_rng(seed)
    n_kps = fixtures.N_KEYPOINTS
    if shape == "linemod":
        K = K_LINEMOD
        lm = fixtures.lm_obj_dict()
        obj_id = sorted(lm.values())[int(rng.integers(0, len(lm)))]   # always drawn: keeps the stream aligned
        if lm_obj_id is not None:
            obj_id = int(lm_obj_id)
        frac = 0.25 if obj_frac is None else obj_frac
        r_px = [np.sqrt(frac * H * W / np.pi)]
        uv = [(W / 2 + rng.uniform(-40, 40), H / 2 + rng.uniform(-15, 15))]
        cls_ids = np.array([1], np.int64)
        mesh = [(fixtures.get_kps(obj_id, ds_type="linemod"), fixtures.get_ctr(obj_id, ds_type="linemod"))]
    elif shape == "ycb":
        K = K_YCB1
        obj_id = None
        n_inst = 5 if n_instances is None else int(n_instances)
        gx, gy = (3, 2) if n_inst <= 6 else (4, 3)
        assert n_inst <= gx * gy
        cells = rng.permutation(gx * gy)[:n_inst]
        cw, ch = W / gx, H / gy
        rmax = min(cw, ch) / 2 - 4
        uv, r_px = [], []
        for cell in cells:
            ix, iy = cell % gx, cell // gx
            if obj_frac is None:
                r = rng.uniform(0.84, 1.0) * rmax
            else:
                r = min(rmax, np.sqrt(obj_frac * H * W / np.pi))
            slack_x, slack_y = cw / 2 - r, ch / 2 - r
            uv.append(((ix + 0.5) * cw + rng.uniform(-slack_x, slack_x), (iy + 0.5) * ch + rng.uniform(-slack_y, slack_y)))
            r_px.append(r)
        cls_ids = np.sort(rng.permutation(np.arange(1, fixtures.YCB_N_CLASSES))[:n_inst]).astype(np.int64)
        mesh = [(fixtures.get_kps(int(c), ds_type="ycb"), fixtures.get_ctr(int(c), ds_type="ycb")) for c in cls_ids]
    else:
        raise ValueError(shape)

    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    centres, radii = [], []
    for (u0, v0), r in zip(uv, r_px):
        z = rng.uniform(0.62, 1.0)
        centres.append(np.array([(u0 - cx) / fx * z, (v0 - cy) / fy * z, z]))
        radii.append(z * r / fx)
    depth, inst = _render(K, centres, radii, rng)
    cld_all = _back_project(depth, K)
    keep = np.sort(rng.choice(H * W, size=n_points, replace=n_points > H * W))   # raster order kept
    pcld = cld_all[keep]
    inst_pt = inst.flatten()[keep]
    labels = np.zeros(n_points, np.int64)
    rgb = rng.uniform(0, 255, size=(n_points, 3)).astype(np.float32)
    nrm = rng.normal(size=(n_points, 3))
    nrm = (nrm / np.linalg.norm(nrm, axis=1, keepdims=True)).astype(np.float32)
    ctr_of = np.zeros((1, n_points, 3), np.float32)
    kp_of = np.zeros((n_kps, n_points, 3), np.float32)
    lo, hi = pcld.min(0), pcld.max(0)
    RTs = np.zeros((len(centres), 3, 4))
    for i, (c, (kps_obj, ctr_obj)) in enumerate(zip(centres, mesh)):
        sel = np.nonzero(inst_pt == i + 1)[0]
        labels[sel] = cls_ids[i]
        R = _haar_rotation(rng)
        t = c - R @ ctr_obj.astype(np.float64)          # object centre sits at the sphere centre
        RTs[i, :, :3], RTs[i, :, 3] = R, t
        targets = np.concatenate((kps_obj.astype(np.float64) @ R.T + t, (R @ ctr_obj + t)[None]), 0)  # [K+1,3]
        votes = targets[:, None, :] + rng.normal(0.0, vote_sigma, size=(n_kps + 1, len(sel), 3))
        n_out = int(round(outlier_frac * len(sel)))
        if n_out:
            out_idx = rng.choice(len(sel), size=n_out, replace=False)
            votes[:, out_idx, :] = rng.uniform(lo, hi, size=(n_kps + 1, n_out, 3))
        p = pcld[sel].astype(np.float64)
        kp_of[:, sel, :] = (p[None] - votes[:n_kps]).astype(np.float32)      # offset = p - kp (ycb_dataset.py:276)
        ctr_of[0, sel, :] = (p - votes[n_kps]).astype(np.float32)
    cld_rgb_nrm = np.concatenate((pcld, rgb, nrm), axis=1).astype(np.float32)
    return Frame(cld_rgb_nrm, pcld.astype(np.float32), labels, ctr_of, kp_of, cls_ids, RTs, obj_id)


def make_batch(shape: str, batch: int, n_points: int = fixtures.N_SAMPLE_POINTS, config_id: int = 2,
               first_frame: int = 0, **kw) -> List[Frame]:
    return [make_frame(shape, n_points, seed=1000 * config_id + first_frame + i, **kw) for i in range(batch)]


def stack(frames: List[Frame]):
    """-> dict of numpy arrays with a leading batch axis (labels as int32 for the kernels)."""
    return {
        "cld_rgb_nrm": np.stack([f.cld_rgb_nrm for f in frames]),
        "pcld": np.stack([f.pcld for f in frames]),
        "labels": np.stack([f.labels for f in frames]).astype(np.int32),
        "ctr_of": np.stack([f.ctr_of[0] for f in frames]),
        "kp_of": np.stack([f.kp_of for f in frames]),
    }


# --------------------------------------------------------------------------------------------------
# ICP refinement inputs: box-like object models, visible surfaces under random poses
# --------------------------------------------------------------------------------------------------
_BOX_NORMALS = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float64)


def box_surface(extents, n: int, rng) -> np.ndarray:
    """n points uniformly on the surface of a box of the given extents centred at the origin -> [n,3] f32"""
    e = np.asarray(extents, np.float64)
    area = np.array([e[1] * e[2]] * 2 + [e[0] * e[2]] * 2 + [e[0] * e[1]] * 2)
    face = rng.choice(6, size=n, p=area / area.sum())
    pts = rng.uniform(-0.5, 0.5, size=(n, 3)) * e
    ax = np.abs(_BOX_NORMALS[face]).argmax(1)
    pts[np.arange(n), ax] = 0.5 * e[ax] * _BOX_NORMALS[face, ax]
    return pts.astype(np.float32)


def visible_box_points(extents, R, t, n: int, noise: float, rng, faces=None) -> np.ndarray:
    """n camera-frame points of the faces of the box (pose R, t) that face a camera at the origin
    (or of the listed face indices), with N(0, noise) per coordinate -> [n,3] f64"""
    e = np.asarray(extents, np.float64)
    if faces is None:
        centres = (0.5 * e * _BOX_NORMALS) @ R.T + t
        faces = [f for f in range(6) if (R @ _BOX_NORMALS[f]) @ centres[f] < 0]
    faces = np.asarray(faces)
    area = np.array([e[1] * e[2]] * 2 + [e[0] * e[2]] * 2 + [e[0] * e[1]] * 2)[faces]
    face = faces[rng.choice(len(faces), size=n, p=area / area.sum())]
    pts = rng.uniform(-0.5, 0.5, size=(n, 3)) * e
    ax = np.abs(_BOX_NORMALS[face]).argmax(1)
    pts[np.arange(n), ax] = 0.5 * e[ax] * _BOX_NORMALS[face, ax]
    return pts @ R.T + t + rng.normal(0.0, noise, size=(n, 3))


def perturb_pose(R, t, angle_deg: float, offset: float, rng):
    """(R', t'): R rotated by angle_deg about a random axis (through the object origin), t moved by
    `offset` metres in a random direction"""
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    a = np.deg2rad(angle_deg)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    dR = np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K
    d = rng.normal(size=3)
    return dR @ R, t + offset * d / np.linalg.norm(d)


def make_icp_batch(batch: int, n_obj: int, pts_per_obj: int, seed: int = 0, n_cls: int = fixtures.YCB_N_CLASSES,
                   model_pts: int = 3000, noise: float = 0.001, outlier_frac: float = 0.0, n_bg: int = 2000,
                   angle_deg: float = 5.0, offset: float = 0.01) -> dict:
    """A batch for IcpRefiner: per-class box-like models (distinct extents, 3-12 cm), and per frame
    n_obj distinct classes, each seen as pts_per_obj points of its camera-facing faces under a random
    pose (z in 0.6-1.0 m) with N(0, noise) noise, `outlier_frac` of them replaced by uniform points in
    the object's bounding box, plus n_bg background-plane points (label 0) at z = 1.2 m; points are
    shuffled.  Returns dict(models: list[n_cls] of [P,3] f32 (None for class 0), extents [n_cls,3],
    pcld [B,N,3] f32, mask [B,N] i32, gt [B,n_cls,3,4] f64, init [B,n_cls,3,4] f32 (gt perturbed by
    angle_deg / offset; identity for absent classes), present [B,n_cls] u8)."""
    rng = np.random.default_rng(seed)
    extents = np.zeros((n_cls, 3))
    models = [None] * n_cls
    for c in range(1, n_cls):
        extents[c] = np.sort(rng.uniform(0.03, 0.12, size=3))[::-1]
        models[c] = box_surface(extents[c], model_pts, rng)
    n = n_obj * pts_per_obj + n_bg
    pcld = np.zeros((batch, n, 3), np.float32)
    mask = np.zeros((batch, n), np.int32)
    gt = np.zeros((batch, n_cls, 3, 4))
    init = np.zeros((batch, n_cls, 3, 4), np.float32)
    init[:, :, :3, :3] = np.eye(3, dtype=np.float32)
    gt[:, :, :3, :3] = np.eye(3)
    present = np.zeros((batch, n_cls), np.uint8)
    grid = [(-0.15, -0.1), (0.0, -0.1), (0.15, -0.1), (-0.15, 0.1), (0.0, 0.1), (0.15, 0.1),
            (-0.3, 0.0), (0.3, 0.0)]
    for b in range(batch):
        cls = np.sort(rng.choice(np.arange(1, n_cls), size=n_obj, replace=False))
        pts, lab = [], []
        for k, c in enumerate(cls):
            R = _haar_rotation(rng)
            gx, gy = grid[k % len(grid)]
            t = np.array([gx, gy, rng.uniform(0.6, 1.0)])
            p = visible_box_points(extents[c], R, t, pts_per_obj, noise, rng)
            n_out = int(round(outlier_frac * pts_per_obj))
            if n_out:
                lo, hi = p.min(0), p.max(0)
                p[rng.choice(pts_per_obj, size=n_out, replace=False)] = rng.uniform(lo, hi, size=(n_out, 3))
            pts.append(p)
            lab.append(np.full(pts_per_obj, c, np.int32))
            gt[b, c, :, :3], gt[b, c, :, 3] = R, t
            Ri, ti = perturb_pose(R, t, angle_deg, offset, rng)
            init[b, c, :, :3], init[b, c, :, 3] = Ri, ti
            present[b, c] = 1
        bg = np.column_stack([rng.uniform(-0.5, 0.5, n_bg), rng.uniform(-0.4, 0.4, n_bg), np.full(n_bg, 1.2)])
        pts.append(bg + rng.normal(0.0, noise, size=(n_bg, 3)))
        lab.append(np.zeros(n_bg, np.int32))
        order = rng.permutation(n)
        pcld[b] = np.concatenate(pts, 0)[order]
        mask[b] = np.concatenate(lab, 0)[order]
    return dict(models=models, extents=extents, pcld=pcld, mask=mask, gt=gt, init=init, present=present)
