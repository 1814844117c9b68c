"""demo.py's pose overlay on the GPU (csrc/vis.cu):

    overlay = PoseOverlay(meshes, device="cuda")                  # packs the class meshes once
    colors = torch.from_numpy(label_colors(n_cls)).to(dev)        # get_label_color(c, n_obj=22, mode=1) per class
    overlay.draw(img, poses, present, cls_ids, K, colors)          # img [B,H,W,3] u8 on the device, drawn in place

    img = draw_p2ds(img, p2ds, r=1, color=(255, 0, 0))             # Basic_Utils.draw_p2ds, numpy in and out

  * PoseOverlay.draw is demo.py:122-145 for a whole batch: every class of a frame's draw order that the frame
    predicted, its mesh moved by the predicted pose, projected (Basic_Utils.project_p3d) and painted point by point as
    a filled disc (Basic_Utils.draw_p2ds); later slots overwrite earlier ones.  A memset and two launches
    (pvn3d_vis_draw_poses), no host sync, so the call can be captured in a CUDA graph.
  * draw_p2ds is the one-call drop-in for Basic_Utils.draw_p2ds on numpy arrays: the image goes to the device, the
    points are clipped (and written back into p2ds, as the reference does) and drawn by the same kernels, and the image
    comes back into the caller's array.
Both take CUDA devices only: there is no CPU fallback.
"""
from __future__ import annotations

import numbers

import numpy as np
import torch

from . import _lib
from ._lib import check, ptr
from .eval_utils import pack_meshes
from .icp import _aligned, _cuda_device

_I32_MIN, _I32_MAX = -2 ** 31, 2 ** 31 - 1


def label_colors(n_cls: int, n_obj: int = 22) -> np.ndarray:
    """[n_cls,3] uint8: row c is Basic_Utils.get_label_color(c, n_obj, mode=1) as cv2 stores it (each channel
    saturated to [0, 255]).  For LineMOD, demo.py colours class 1 with get_label_color(obj_id): put that row there."""
    c = np.arange(int(n_cls), dtype=np.int64)
    m = 255 * 255 * 255 // int(n_obj) * c
    return np.clip(np.stack([m // 255 // 255, (m // 255) % 255, m % 255], 1), 0, 255).astype(np.uint8)


def cv_color(color) -> tuple:
    """the three uint8 channels cv2.circle paints for `color` on a 3-channel image: missing channels are 0, each value
    is rounded half to even and saturated to [0, 255]; NaN, infinities and values outside int32 become 0 (cvRound's
    x86-64 result, INT_MIN, saturated)"""
    vals = [float(v) for v in np.asarray(color, dtype=np.float64).reshape(-1)[:3]]
    out = []
    for v in vals + [0.0] * (3 - len(vals)):
        q = np.rint(v)
        out.append(0 if not (_I32_MIN <= q <= _I32_MAX) else int(min(max(q, 0), 255)))
    return tuple(out)


def _is_color(color) -> bool:
    try:
        a = np.asarray(color)
    except Exception:
        return False
    return a.ndim <= 1 and 1 <= a.size <= 4 and (a.dtype.kind in "iuf" or a.dtype == np.bool_)


def _is_radius(r) -> bool:
    return isinstance(r, (numbers.Integral, np.integer)) and not isinstance(r, (bool, np.bool_))


def gpu_drawable(img, p2ds, r=1, color=(255, 0, 0)) -> bool:
    """whether draw_p2ds takes this call: a C-contiguous uint8 [H,W,3] ndarray, int32 / int64 [n,2] points, an integer
    r >= 0, a colour of 1 to 4 real numbers, and a CUDA device"""
    return (isinstance(img, np.ndarray) and img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3
            and img.flags.c_contiguous and img.flags.writeable and img.shape[0] > 0 and img.shape[1] > 0
            and isinstance(p2ds, np.ndarray) and p2ds.dtype in (np.int32, np.int64) and p2ds.ndim == 2
            and p2ds.shape[1] == 2 and p2ds.flags.writeable and _is_radius(r) and int(r) >= 0 and _is_color(color)
            and torch.cuda.is_available())


_WS = {}   # device -> (owner, address, bytes): the drop-in's stamp plane


def _workspace(cache: dict, key, nbytes: int, dev):
    hit = cache.get(key)
    if hit is None or hit[2] < nbytes:
        owner, addr = _aligned(nbytes, dev)
        hit = cache[key] = (owner, addr, nbytes)
    return hit


def draw_p2ds(img: np.ndarray, p2ds: np.ndarray, r: int = 1, color=(255, 0, 0)) -> np.ndarray:
    """Basic_Utils.draw_p2ds (basic_utils.py:315-323) on the current CUDA device: p2ds is clipped in place to [0, w] x
    [0, h], every point paints cv2.circle(img, p, r, color, -1) into img in place, and img itself is returned."""
    if not (isinstance(img, np.ndarray) and img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3
            and img.flags.c_contiguous):
        raise TypeError("draw_p2ds: img must be a C-contiguous uint8 [H,W,3] ndarray")
    if not (isinstance(p2ds, np.ndarray) and p2ds.dtype in (np.int32, np.int64) and p2ds.ndim == 2
            and p2ds.shape[1] == 2):
        raise TypeError("draw_p2ds: p2ds must be an int32 or int64 [n,2] ndarray")
    if not _is_radius(r) or int(r) < 0:
        raise ValueError(f"draw_p2ds: r must be an integer >= 0, got {r!r}")
    if not _is_color(color):
        raise ValueError(f"draw_p2ds: color must be 1 to 4 real numbers, got {color!r}")
    c0, c1, c2 = cv_color(color)
    h, w = img.shape[:2]
    if p2ds.shape[0] == 0:
        return img
    dev = _cuda_device("cuda", "draw_p2ds")
    lib = _lib.load()
    q = p2ds if p2ds.dtype == np.int32 else np.clip(p2ds, _I32_MIN, _I32_MAX).astype(np.int32)
    t_img = torch.from_numpy(img).to(dev)
    t_p = torch.from_numpy(np.ascontiguousarray(q)).to(dev)
    nbytes = int(lib.pvn3d_vis_workspace_bytes(1, h, w))
    _, ws, ws_bytes = _workspace(_WS, dev, nbytes, dev)
    with torch.cuda.device(dev):
        rc = lib.pvn3d_vis_draw_p2ds(ptr(t_img), h, w, ptr(t_p), int(p2ds.shape[0]), int(r), c0 | c1 << 8 | c2 << 16,
                                     ws, ws_bytes, torch.cuda.current_stream(dev).cuda_stream)
    check(rc, "pvn3d_vis_draw_p2ds")
    torch.from_numpy(img).copy_(t_img)
    p2ds[...] = t_p.cpu().numpy()
    return img


def _dev_tensor(t, dev, what):
    if not torch.is_tensor(t) or t.device != dev:
        raise ValueError(f"PoseOverlay.draw: {what} must be a tensor on {dev}")
    return t


class PoseOverlay:
    """Draw predicted poses onto a batch of frames, as demo.py draws one frame.

    meshes: {class id: [P,3]} or a list indexed by class id (entry 0 ignored); every class 1 .. n_cls-1 needs points
    (eval_utils.pack_meshes).  n_cls = largest id + 1 must equal the pose table's second dimension."""

    def __init__(self, meshes, device="cuda"):
        self.dev = _cuda_device(device, "PoseOverlay")
        pts, off = pack_meshes(meshes)
        self.n_cls = off.size - 1
        self.max_pts = int(np.diff(off)[1:].max())
        self.meshes = torch.from_numpy(pts).to(self.dev)
        self.mesh_off = torch.from_numpy(off).to(self.dev)
        self.lib = _lib.load()
        self._ws = {}

    def draw(self, img: torch.Tensor, poses: torch.Tensor, present: torch.Tensor, order: torch.Tensor, K: torch.Tensor,
             colors: torch.Tensor, radius: int = 1, cam_scale: float = 1.0) -> torch.Tensor:
        """Draw into img [B,H,W,3] uint8 (C-contiguous) in place and return it.  All tensors on this overlay's device:
        poses [B,n_cls,3,4] float32 or float64; present [B,n_cls] (bool or integer, nonzero = predicted); order [B,S]
        or [B,S,1] class ids in draw order (demo.py's cls_ids; 0 and ids outside [1, n_cls) are skipped); K [3,3] or
        [B,3,3]; colors [n_cls,3] uint8.  No host sync."""
        dev = self.dev
        _dev_tensor(img, dev, "img")
        if img.dtype != torch.uint8 or img.dim() != 4 or img.shape[3] != 3 or not img.is_contiguous():
            raise ValueError(f"PoseOverlay.draw: img must be C-contiguous uint8 [B,H,W,3], got {img.dtype} "
                             f"{tuple(img.shape)}")
        b, h, w = (int(x) for x in img.shape[:3])
        _dev_tensor(poses, dev, "poses")
        if poses.dtype not in (torch.float32, torch.float64) or tuple(poses.shape[:1]) + tuple(poses.shape[2:]) != (b, 3, 4) \
                or poses.dim() != 4:
            raise ValueError(f"PoseOverlay.draw: poses must be float32 / float64 [{b},n_cls,3,4], got {poses.dtype} "
                             f"{tuple(poses.shape)}")
        if poses.shape[1] != self.n_cls:
            raise ValueError(f"PoseOverlay.draw: pose table has {poses.shape[1]} classes, the meshes {self.n_cls}")
        _dev_tensor(present, dev, "present")
        if present.numel() != b * self.n_cls or present.is_floating_point():
            raise ValueError(f"PoseOverlay.draw: present must be bool / integer [{b},{self.n_cls}]")
        _dev_tensor(order, dev, "order")
        if order.is_floating_point() or order.dtype == torch.bool or order.dim() not in (2, 3) or order.shape[0] != b \
                or (order.dim() == 3 and order.shape[2] != 1) or order.shape[1] < 1:
            raise ValueError(f"PoseOverlay.draw: order must be integer [{b},S] or [{b},S,1], got {order.dtype} "
                             f"{tuple(order.shape)}")
        s = int(order.shape[1])
        _dev_tensor(K, dev, "K")
        if not K.is_floating_point() or tuple(K.shape[-2:]) != (3, 3) or K.dim() not in (2, 3) \
                or (K.dim() == 3 and K.shape[0] != b):
            raise ValueError(f"PoseOverlay.draw: K must be float [3,3] or [{b},3,3], got {tuple(K.shape)}")
        _dev_tensor(colors, dev, "colors")
        if colors.dtype != torch.uint8 or tuple(colors.shape) != (self.n_cls, 3):
            raise ValueError(f"PoseOverlay.draw: colors must be uint8 [{self.n_cls},3], got {colors.dtype} "
                             f"{tuple(colors.shape)}")
        if not _is_radius(radius) or int(radius) < 0:
            raise ValueError(f"PoseOverlay.draw: radius must be an integer >= 0, got {radius!r}")
        ps = poses.contiguous()
        pr = (present.reshape(b, self.n_cls) != 0).to(torch.uint8).contiguous()
        od = order.reshape(b, s).to(torch.int32).contiguous()
        kk = K.to(torch.float64).expand(b, 3, 3).contiguous()
        col = colors.contiguous()
        nbytes = int(self.lib.pvn3d_vis_workspace_bytes(b, h, w))
        _, ws, ws_bytes = _workspace(self._ws, None, nbytes, dev)
        with torch.cuda.device(dev):
            rc = self.lib.pvn3d_vis_draw_poses(ptr(img), b, h, w, ptr(self.meshes), ptr(self.mesh_off), self.n_cls,
                                               self.max_pts, ptr(ps), int(ps.dtype == torch.float64), ptr(pr), ptr(od),
                                               s, ptr(kk), float(cam_scale), ptr(col), int(radius), ws, ws_bytes,
                                               torch.cuda.current_stream(dev).cuda_stream)
        check(rc, "pvn3d_vis_draw_poses")
        return img
