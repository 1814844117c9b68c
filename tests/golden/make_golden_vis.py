"""Record demo.py's pose overlay from the REFERENCE ITSELF on the CPU (build container only).

    python tests/golden/make_golden_vis.py          # writes vis_cases.npz + make_golden_vis.log

The unmodified Basic_Utils (project_p3d, draw_p2ds, get_label_color) composed as demo.py:122-145 composes them: for each
class of a frame's cls_ids that the frame predicted, mesh_pts = np.dot(mesh, pose[:, :3].T) + pose[:, 3] in float64,
project_p3d(mesh_pts, cam_scale, K), draw_p2ds(img, p2ds, r, color).  Seeded synthetic frames (a uniform-noise
background from vis_ref.background(seed), so every painted pixel is seen):

  ov0_ycb     2 frames 480x640, ycb_K1, 22 classes with synthetic meshes, 22 zero-padded slots, 5 overlapping objects per
              frame, one listed class not predicted and one predicted class not listed; colours get_label_color(c, 22, 1)
  ov1_lm      1 frame, the linemod K, one 2000-point object, colour get_label_color(obj_id) in row 1, cls_ids [1, 0]
  ov2..ov6    edge frames at r = 0, 1, 3, 4, 7: points behind the camera, at z = 0, z < 1e-8 and just above it
              (projections beyond int32), points off every border, a NaN pose, a class listed twice, an object cut by
              the border; colours out of range and non-integer
  dp0..dp4    Basic_Utils.draw_p2ds alone on integer points: INT_MIN / INT_MAX, negative, exactly w and h, r 0 .. 7,
              colours of 1, 3 and 4 channels, out of range, non-integer, NaN and beyond int32; one 37x53 image

Recorded per case: its inputs, each output image as a SHA-256 plus its changed pixels (flat index, value), and the
clipped p2ds (the overlay cases: of every drawn slot, in draw order).  Poses are float32-representable float64, so the
GPU test can also pass them as float32.  While recording, tests/vis_ref.py is checked against every reference output
bit for bit, and the projected coordinates within 1e-9 px of a .5 tie are counted; a mismatch aborts.
"""
import os
import sys
import time
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
REF = os.environ.get("PVN3D_REFERENCE", "/root/reference/pvn3d")

from pvn3d_b200 import compat, synth  # noqa: E402
from oracle import ext_cpu  # noqa: E402
import vis_ref as V  # noqa: E402

if not hasattr(np, "bool"):
    np.bool = bool  # the reference's ip_basic predates numpy 1.24
compat.install_import_shims()
sys.modules["lib.pointnet2_utils._ext"] = ext_cpu
sys.path.insert(0, REF)
LOG = []


def log(msg):
    print(msg)
    LOG.append(msg)


def _mesh(rng, n, size):
    """n float32 points on an ellipsoid shell with semi-axes `size` (metres)"""
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return (d * size * rng.uniform(0.8, 1.0, (n, 1))).astype(np.float32)


def _pose(rng, t):
    r = synth._haar_rotation(rng)
    return np.concatenate([r, np.asarray(t, np.float64)[:, None]], 1).astype(np.float32).astype(np.float64)


def _pack(meshes, n_cls):
    off = [0]
    for c in range(1, n_cls):
        off.append(off[-1] + len(meshes[c]))
    return np.concatenate([meshes[c] for c in range(1, n_cls)], 0), np.asarray([0] + off, np.int32)


def ycb_case(rng, K):
    n_cls, slots = 22, 22
    meshes = {c: _mesh(rng, int(rng.integers(300, 900)), rng.uniform(0.03, 0.07, 3)) for c in range(1, n_cls)}
    frames = [([2, 5, 9, 14, 20], 9, 11), ([21, 1, 6, 5, 13], 6, 3)]   # (cls_ids, listed not predicted, predicted unlisted)
    poses = np.zeros((2, n_cls, 3, 4))
    present = np.zeros((2, n_cls), np.uint8)
    order = np.zeros((2, slots), np.int32)
    for f, (ids, missing, extra) in enumerate(frames):
        order[f, :len(ids)] = ids
        for j, c in enumerate(ids + [extra]):
            poses[f, c] = _pose(rng, [-0.08 + 0.04 * j + rng.uniform(-0.01, 0.01), rng.uniform(-0.04, 0.04),
                                      rng.uniform(0.75, 0.95)])
            present[f, c] = c != missing
    colors = np.array([bu.get_label_color(c, n_obj=22, mode=1) for c in range(n_cls)], np.float64)
    return dict(meshes=meshes, n_cls=n_cls, poses=poses, present=present, order=order, K=np.stack([K, K]),
                colors=colors, r=1, cam_scale=1.0, h=480, w=640)


def lm_case(rng, K, obj_id=4):
    meshes = {1: _mesh(rng, 2000, np.array([0.05, 0.04, 0.06]))}
    poses = np.zeros((1, 2, 3, 4))
    poses[0, 1] = _pose(rng, [0.02, -0.01, 0.7])
    colors = np.zeros((2, 3))
    colors[1] = bu.get_label_color(obj_id, n_obj=22, mode=1)
    return dict(meshes=meshes, n_cls=2, poses=poses, present=np.array([[0, 1]], np.uint8),
                order=np.array([[1, 0]], np.int32), K=K[None], colors=colors, r=1, cam_scale=1.0, h=480, w=640)


def edge_case(rng, K, r):
    n_cls = 5
    eye = np.concatenate([np.eye(3), np.zeros((3, 1))], 1)
    # class 1: in the camera frame (identity pose): behind the camera, z = 0, z < 1e-8, z just above 1e-8 (x / z far
    # beyond int32), and a few ordinary points
    z = np.array([-0.5, -1e-3, 0.0, 5e-9, -0.0, 2e-8, 1e-7, 3e-8, 0.8, 0.9, 1.1, 0.7], np.float32)
    x = np.array([0.1, -0.2, 0.05, -0.05, 0.3, 0.5, -0.4, 0.0, 0.01, -0.02, 0.03, 0.2], np.float32)
    y = np.array([-0.1, 0.2, 0.05, 0.01, -0.3, -0.5, 0.4, 1e-3, 0.02, -0.01, 0.0, -0.15], np.float32)
    m1 = np.stack([x, y, z], 1)
    # class 2: off every border and exactly on it after rounding; x, y in pixels -> camera frame at z = 1
    px = np.array([-50, 700, 320, 320, -10, 650, 640, 0, 639.5, 640.4, 320, -0.5, 300], np.float64)
    py = np.array([240, 240, -40, 520, -10, 490, 480, 0, 479.5, 100, 480.6, 200, -0.6], np.float64)
    kk = K.astype(np.float64)
    m2 = np.stack([(px - kk[0, 2]) / kk[0, 0], (py - kk[1, 2]) / kk[1, 1], np.ones_like(px)], 1).astype(np.float32)
    m3 = _mesh(rng, 40, np.array([0.03, 0.03, 0.03]))        # drawn with a NaN pose
    m4 = _mesh(rng, 120, np.array([0.06, 0.05, 0.04]))       # an object cut by the right border, listed twice
    poses = np.zeros((1, n_cls, 3, 4))
    poses[0, 1] = eye
    poses[0, 2] = eye
    poses[0, 3] = _pose(rng, [0.0, 0.0, 0.8])
    poses[0, 3, 1, 2] = np.nan
    poses[0, 4] = _pose(rng, [0.27, 0.05, 0.9])
    colors = np.array([[0, 0, 0], [300.6, -3, 2.5], [0.5, 1.5, 254.5], [255.5, 127.5, -0.5], [12.4, 3e9, 99.5]])
    return dict(meshes={1: m1, 2: m2, 3: m3, 4: m4}, n_cls=n_cls, poses=poses, present=np.array([[0, 1, 1, 1, 1]], np.uint8),
                order=np.array([[4, 1, 2, 3, 0, 4]], np.int32), K=K[None], colors=colors, r=r,
                cam_scale=1.0 if r != 4 else 1.25, h=480, w=640)


def reference_overlay(case, seeds):
    """demo.py's loop with the reference's own helpers, one frame at a time"""
    outs, p2ds = [], []
    for f in range(len(seeds)):
        img = V.background(seeds[f], case["h"], case["w"])
        pred_cls_ids = np.nonzero(case["present"][f])[0]
        for cls_id in case["order"][f]:
            idx = np.where(pred_cls_ids == cls_id)[0]
            if cls_id == 0 or len(idx) == 0:
                continue
            pose = case["poses"][f, cls_id]
            mesh_pts = case["meshes"][cls_id].copy()
            with np.errstate(invalid="ignore"):
                mesh_pts = np.dot(mesh_pts, pose[:, :3].T) + pose[:, 3]
                mp = bu.project_p3d(mesh_pts, case["cam_scale"], case["K"][f])
            color = tuple(float(v) for v in case["colors"][cls_id])
            img = bu.draw_p2ds(img, mp, r=case["r"], color=color)
            p2ds.append(mp)
        outs.append(img)
    return outs, p2ds


def restated_overlay(case, seeds):
    outs, p2ds = [], []
    for f in range(len(seeds)):
        img, drawn = V.overlay_frame(V.background(seeds[f], case["h"], case["w"]), case["meshes"], case["poses"][f],
                                     case["present"][f], case["order"][f], case["K"][f], case["colors"], case["r"],
                                     case["cam_scale"])
        outs.append(img)
        p2ds += drawn
    return outs, p2ds


def record_images(out, key, seeds, imgs, h, w):
    idx, vals, cnt = [], [], []
    for s, img in zip(seeds, imgs):
        i, v = V.changed(V.background(s, h, w), img)
        idx.append(i)
        vals.append(v)
        cnt.append(len(i))
    out[key + "sha"] = np.stack([np.frombuffer(V.sha(img), np.uint8) for img in imgs])
    out[key + "chg_idx"] = np.concatenate(idx)
    out[key + "chg_val"] = np.concatenate(vals)
    out[key + "chg_cnt"] = np.asarray(cnt, np.int64)
    return cnt


def main():
    global bu
    from lib.utils import basic_utils as bu_mod

    bu = bu_mod.Basic_Utils(types.SimpleNamespace(dataset_name="linemod"))
    import cv2

    t0 = time.time()
    log(f"reference {REF}, cv2 {cv2.__version__}, numpy {np.__version__}")
    K_ycb = bu_mod.intrinsic_matrix["ycb_K1"].astype(np.float64)
    K_lm = bu_mod.intrinsic_matrix["linemod"].astype(np.float64)
    rng = np.random.default_rng(20261017)
    cases = [("ycb", ycb_case(rng, K_ycb)), ("lm", lm_case(rng, K_lm))]
    cases += [(f"edge_r{r}", edge_case(rng, K_ycb, r)) for r in (0, 1, 3, 4, 7)]
    out = {"n_overlay": np.int64(len(cases))}
    ties = 0
    for i, (name, c) in enumerate(cases):
        k = f"ov{i}_"
        b = c["poses"].shape[0]
        seeds = [1000 * i + f for f in range(b)]
        ref_imgs, ref_p2ds = reference_overlay(c, seeds)
        my_imgs, my_p2ds = restated_overlay(c, seeds)
        assert all(np.array_equal(a, m) for a, m in zip(ref_imgs, my_imgs)), f"{name}: vis_ref image differs"
        ref_p2ds = [V.clip(p, c["h"], c["w"]) for p in ref_p2ds]   # draw_p2ds clipped them in place already
        assert len(ref_p2ds) == len(my_p2ds) and all(np.array_equal(a, m) for a, m in zip(ref_p2ds, my_p2ds)), name
        for f in range(b):
            for cls in c["order"][f]:
                if 1 <= cls < c["n_cls"] and c["present"][f, cls]:
                    ties += V.near_ties(V.project_raw(V.transform(c["meshes"][cls], c["poses"][f, cls]),
                                                      c["cam_scale"], c["K"][f]))
        pts, off = _pack(c["meshes"], c["n_cls"])
        out.update({k + "name": np.array(name), k + "mesh_pts": pts, k + "mesh_off": off, k + "poses": c["poses"],
                    k + "present": c["present"], k + "order": c["order"], k + "K": c["K"], k + "colors": c["colors"],
                    k + "r": np.int64(c["r"]), k + "cam_scale": np.float64(c["cam_scale"]), k + "hw": np.array([c["h"], c["w"]]),
                    k + "seeds": np.asarray(seeds, np.int64), k + "p2ds": np.concatenate(ref_p2ds).astype(np.int32),
                    k + "p2ds_cnt": np.asarray([len(p) for p in ref_p2ds], np.int64)})
        cnt = record_images(out, k, seeds, ref_imgs, c["h"], c["w"])
        log(f"{k}{name}: {b} frame(s), {len(ref_p2ds)} drawn slots, {sum(len(p) for p in ref_p2ds)} points, r={c['r']}, "
            f"changed pixels {cnt}; vis_ref bit-equal")
    # draw_p2ds alone
    big = np.array([[-2 ** 31, 5], [2 ** 31 - 1, 2 ** 31 - 1], [-7, -9], [640, 480], [639, 479], [0, 0], [640, 0],
                    [0, 480], [320, -2 ** 31], [700, 200], [-1, 481]], np.int32)
    lm_p2ds = V.project(V.transform(cases[1][1]["meshes"][1], cases[1][1]["poses"][0, 1]), 1.0, K_lm)
    rnd = rng.integers(-30, 700, (300, 2)).astype(np.int32)
    dps = [(480, 640, lm_p2ds, 1, (255, 0, 0)), (480, 640, np.concatenate([big, rnd]), 4, (300.6, -3, 2.5)),
           (480, 640, np.concatenate([big, rnd[:50]]), 0, (0.5, 1.5, 254.5, 99)),
           (37, 53, rng.integers(-10, 64, (60, 2)).astype(np.int32), 7, (2.5,)),
           (480, 640, np.concatenate([big, rnd[50:120]]), 3, (1e10, float("nan"), -7.5))]
    out["n_p2ds"] = np.int64(len(dps))
    for i, (h, w, p, r, color) in enumerate(dps):
        k = f"dp{i}_"
        seed = 5000 + i
        img = V.background(seed, h, w)
        p_ref = p.copy()
        res = bu.draw_p2ds(img, p_ref, r=r, color=color)
        assert res is img
        mine = V.draw(V.background(seed, h, w), V.clip(p, h, w), r, color)
        assert np.array_equal(mine, img) and np.array_equal(V.clip(p, h, w), p_ref), f"draw_p2ds case {i}: vis_ref differs"
        out.update({k + "hw": np.array([h, w]), k + "p2ds_in": p, k + "p2ds_out": p_ref, k + "r": np.int64(r),
                    k + "color": np.asarray(color, np.float64), k + "seeds": np.array([seed], np.int64)})
        cnt = record_images(out, k, [seed], [img], h, w)
        log(f"{k}: {h}x{w}, {len(p)} points, r={r}, color={color}, changed pixels {cnt[0]}; vis_ref bit-equal")
    log(f"projected coordinates within 1e-9 px of a .5 tie: {ties}")
    assert ties == 0, "a projected coordinate lies on a rounding tie: the dot-product order would decide it"
    path = os.path.join(HERE, "vis_cases.npz")
    np.savez_compressed(path, **out)
    log(f"vis_cases.npz {os.path.getsize(path) / 1e6:.2f} MB, recorded in {time.time() - t0:.1f} s")
    with open(os.path.join(HERE, "make_golden_vis.log"), "w") as f:
        f.write("\n".join(LOG) + "\n")


if __name__ == "__main__":
    main()
