"""ICP pose refinement -- the reference's `my_icp` (lib/utils/icp/icp.py:141-192), run on the GPU in
float64 by csrc/icp.cu.

    T, distances, i = my_icp(A, B, init_pose, max_iterations=500, tolerance=1e-9)   # drop-in, one object
    ref = IcpRefiner(models, n_cls, batch, n_pts, max_pts=..., min_pts=..., device="cuda")
    poses64, iters, err, refined = ref.refine(pcld, mask, poses, present)          # batched, sync-free
    p3ds = get_cld_bigest_clus(p3ds, radius=0.06)    # eval_icp's biggest flat mean-shift cluster
    ref = IcpRefiner(..., cluster_bandwidth=0.06)    # the same filter before every batched fit
    ref = DepthIcpRefiner(models, n_cls, batch)      # eval_icp's settings on full-resolution depth
    poses64, iters, err, refined = ref.refine(depth, K, cam_scale, poses, present, pcld=pcld, point_labels=mask)

The batched form takes FramePoseSolver.solve()'s poses and present flags as they come out and runs
one fit per (frame, class) on the current stream, as pvn3d/eval_icp.py:94-185 does per object.
"""
from __future__ import annotations

from typing import Dict, Sequence, Union

import numpy as np
import torch

from . import _lib
from ._lib import check, ptr

_ALIGN = 256


def _aligned(nbytes: int, dev) -> tuple:
    """(owner tensor, 256-byte aligned device address) of a scratch buffer"""
    buf = torch.empty((max(int(nbytes), 1) + _ALIGN,), dtype=torch.uint8, device=dev)
    return buf, (buf.data_ptr() + _ALIGN - 1) // _ALIGN * _ALIGN


def _cuda_device(device, who: str) -> torch.device:
    """torch.device with an explicit index ("cuda" -> the current device), so that it compares equal
    to a tensor's .device"""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError(f"{who}: CUDA only -- no CPU fallback")
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    return dev


def _points(x, name: str) -> np.ndarray:
    a = x.detach().cpu().numpy() if torch.is_tensor(x) else np.asarray(x)
    a = np.ascontiguousarray(a, dtype=np.float32)
    if a.ndim != 2 or a.shape[1] != 3:
        raise ValueError(f"{name}: expected [P,3] points, got shape {a.shape}")
    return a


def model_table(models: Union[Sequence, Dict[int, object]], n_cls: int):
    """Per-class model points -> (pts [total,3] f32, model_off [n_cls+1] i32).  Class 0 and classes
    without a model get an empty range (never refined)."""
    n_cls = int(n_cls)
    if isinstance(models, dict):
        items = {int(k): v for k, v in models.items()}
    else:
        items = {c: v for c, v in enumerate(models)}
    bad = [c for c in items if not 0 <= c < n_cls]
    if bad:
        raise ValueError(f"model class ids {bad} outside [0, {n_cls})")
    pts, off = [], [0]
    for c in range(n_cls):
        v = items.get(c)
        a = np.zeros((0, 3), np.float32) if (c == 0 or v is None) else _points(v, f"models[{c}]")
        pts.append(a)
        off.append(off[-1] + len(a))
    return np.concatenate(pts, 0), np.asarray(off, np.int32)


class IcpModels:
    """Device-side nearest-neighbour structure of a set of object-frame models (built on the GPU).
    The build runs on the current stream; `ready` is recorded after it, and every user of the
    structure on another stream waits for that event first."""

    def __init__(self, pts: np.ndarray, model_off: np.ndarray, device):
        self.lib = _lib.load()
        self.dev = _cuda_device(device, "IcpModels")
        self.n_models, self.total = len(model_off) - 1, int(model_off[-1])
        nbytes = int(self.lib.pvn3d_icp_models_bytes(self.n_models, self.total))
        if nbytes == 0:
            raise ValueError("IcpModels: empty model set")
        self._buf, self.ptr = _aligned(nbytes, self.dev)
        self.nbytes = nbytes
        d_pts = torch.from_numpy(np.ascontiguousarray(pts, np.float32).reshape(-1, 3)).to(self.dev)
        d_off = torch.from_numpy(np.ascontiguousarray(model_off, np.int32)).to(self.dev)
        with torch.cuda.device(self.dev):
            st = torch.cuda.current_stream(self.dev)
            rc = self.lib.pvn3d_icp_build_models(ptr(d_pts) if self.total else 0, ptr(d_off), self.n_models,
                                                 self.total, self.ptr, nbytes, st.cuda_stream)
        check(rc, "pvn3d_icp_build_models")
        d_pts.record_stream(st)
        d_off.record_stream(st)
        self.ready = torch.cuda.Event()
        self.ready.record(st)


class IcpRefiner:
    """Batched ICP refinement of the solver's poses for a fixed (batch, n_pts, n_cls) shape.

    models   per-class object-frame points: a list indexed by class id or a {class id: [P_c,3]} dict;
             class 0 is unused, and a class without a model is never refined.
    max_pts  scene points per fit: a class with more points in the mask keeps max_pts of them, at
             positions floor(j * cnt / max_pts) of its points in ascending index (deterministic; the
             reference draws a random subset).
    min_pts  a class with fewer points in the mask is not refined (its pose passes through).
    Both are required.  pvn3d/eval_icp.py uses max_pts=2000, min_pts=1500, counted on full-resolution
    depth masks; a network cloud of 12288 points holds only about 1000-1300 points per YCB-sized
    object, so those values would skip every fit there: choose them for the cloud at hand.
    max_iter, tol  eval_icp's 500 and 1e-9 (my_icp's own defaults are 20 and 1e-3).
    cluster_bandwidth  None (default): fit every selected point.  A bandwidth (eval_icp uses 0.06): first
             keep only the biggest cluster of sklearn's flat MeanShift(bandwidth, bin_seeding=True,
             max_iter=cluster_max_iter) of each fit's selection, as eval_icp's get_cld_bigest_clus does,
             and fit those points; `cluster_pts` [B,n_cls] i32 then holds how many each fit used
             (0 when skipped).  Needs max_pts <= 4096.
    """

    def __init__(self, models, n_cls: int, batch: int, n_pts: int, *, max_pts: int, min_pts: int,
                 max_iter: int = 500, tol: float = 1e-9, cluster_bandwidth=None, cluster_max_iter: int = 300,
                 device="cuda"):
        self.dev = _cuda_device(device, "IcpRefiner")
        self.n_cls, self.b, self.n = int(n_cls), int(batch), int(n_pts)
        self.max_pts, self.min_pts = int(max_pts), int(min_pts)
        self.max_iter, self.tol = int(max_iter), float(tol)
        if not 2 <= self.n_cls <= 64:
            raise ValueError(f"n_cls={n_cls}: 2..64 classes")
        if self.b < 1 or self.n < 1:
            raise ValueError(f"batch={batch}, n_pts={n_pts}: both must be >= 1")
        if self.max_pts < 1 or self.min_pts < 0:
            raise ValueError(f"max_pts={max_pts} must be >= 1 and min_pts={min_pts} >= 0")
        if self.max_iter < 1 or not self.tol >= 0.0:
            raise ValueError(f"max_iter={max_iter} must be >= 1 and tol={tol} >= 0")
        self.cluster_bw = None if cluster_bandwidth is None else float(cluster_bandwidth)
        self.cluster_max_iter = int(cluster_max_iter)
        if self.cluster_bw is not None:
            if not 0.0 < self.cluster_bw < float("inf") or self.cluster_max_iter < 0:
                raise ValueError(f"cluster_bandwidth={cluster_bandwidth} must be > 0 and finite, "
                                 f"cluster_max_iter={cluster_max_iter} >= 0")
            if self.max_pts > _lib.FLAT_MS_MAX_PTS:
                raise ValueError(f"max_pts={max_pts}: the cluster filter takes at most {_lib.FLAT_MS_MAX_PTS} "
                                 "points per fit")
        pts, off = model_table(models, self.n_cls)
        self.lib = _lib.load()
        self.models = IcpModels(pts, off, self.dev)
        ws_query = (self.lib.pvn3d_icp_workspace_bytes if self.cluster_bw is None
                    else self.lib.pvn3d_icp_clustered_workspace_bytes)
        self.ws_bytes = int(ws_query(self.b, self.n, self.n_cls, self.max_pts))
        if self.ws_bytes == 0:
            raise ValueError("IcpRefiner: problem too large for 32-bit indexing")
        self._ws, self._ws_ptr = _aligned(self.ws_bytes, self.dev)
        shape = (self.b, self.n_cls)
        self.poses = torch.empty(shape + (3, 4), dtype=torch.float64, device=self.dev)
        self.iters = torch.empty(shape, dtype=torch.int32, device=self.dev)
        self.err = torch.empty(shape, dtype=torch.float64, device=self.dev)
        self.refined = torch.empty(shape, dtype=torch.uint8, device=self.dev)
        #: points each fit of the last refine() used after the cluster filter (cluster_bandwidth set only)
        self.cluster_pts = None if self.cluster_bw is None else torch.empty(shape, dtype=torch.int32, device=self.dev)

    def pair_tests(self) -> int:
        """diagnostics (synchronises): model points the last refine()'s searches tested"""
        off = self._ws_ptr - self._ws.data_ptr()
        return int(self._ws[off:off + 8].view(torch.int64).item())

    def kept_points(self) -> torch.Tensor:
        """cluster filter only: [B,N] int32 device view of the workspace.  After refine(), row b holds,
        for each refined class c, the cluster_pts[b, c] frame point indices (into pcld[b]) that fit (b, c)
        used, ascending, starting at position (number of points of frame b with class id in 1..c-1); the
        rest is unspecified.  Valid until the next refine() on the same stream."""
        if self.cluster_bw is None:
            raise RuntimeError("IcpRefiner.kept_points: the refiner has no cluster filter")
        off = self._ws_ptr - self._ws.data_ptr() + int(self.lib.pvn3d_icp_workspace_bytes(self.b, self.n, self.n_cls,
                                                                                          self.max_pts))
        return self._ws[off:off + 4 * self.b * self.n].view(torch.int32).view(self.b, self.n)

    def refine(self, pcld: torch.Tensor, mask: torch.Tensor, poses: torch.Tensor, present: torch.Tensor):
        """pcld [B,N,3] f32, mask [B,N] i32 (the solver's new_mask for YCB, the network mask for LineMOD),
        poses [B,n_cls,3,4] f32 and present [B,n_cls] u8 from FramePoseSolver.solve().  Returns
        (poses [B,n_cls,3,4] f64, iters [B,n_cls] i32, err [B,n_cls] f64, refined [B,n_cls] u8): views
        of refiner-owned buffers, valid until the next refine() on the same stream.  No host sync."""
        b = pcld.size(0)
        if not (1 <= b <= self.b and pcld.shape[1:] == (self.n, 3) and mask.shape == (b, self.n)
                and poses.shape == (b, self.n_cls, 3, 4) and present.shape == (b, self.n_cls)):
            raise ValueError("IcpRefiner.refine: shapes do not match the refiner")
        for t, dt in ((pcld, torch.float32), (mask, torch.int32), (poses, torch.float32), (present, torch.uint8)):
            if not (t.is_cuda and t.is_contiguous() and t.dtype == dt and t.device == self.dev):
                raise ValueError(f"IcpRefiner.refine: expected contiguous {dt} on {self.dev}")
        with torch.cuda.device(self.dev):
            cur = torch.cuda.current_stream(self.dev)
            cur.wait_event(self.models.ready)                 # the model build may have run on another stream
            if self.cluster_bw is None:
                rc = self.lib.pvn3d_icp_refine_batch(
                    self.models.ptr, ptr(pcld), ptr(mask), b, self.n, self.n_cls, ptr(poses), ptr(present),
                    self.max_pts, self.min_pts, self.max_iter, self.tol, ptr(self.poses), ptr(self.iters),
                    ptr(self.err), ptr(self.refined), self._ws_ptr, self.ws_bytes,
                    cur.cuda_stream)
            else:
                rc = self.lib.pvn3d_icp_refine_batch_clustered(
                    self.models.ptr, ptr(pcld), ptr(mask), b, self.n, self.n_cls, ptr(poses), ptr(present),
                    self.max_pts, self.min_pts, self.max_iter, self.tol, self.cluster_bw, self.cluster_max_iter,
                    ptr(self.poses), ptr(self.iters), ptr(self.err), ptr(self.refined), ptr(self.cluster_pts),
                    self._ws_ptr, self.ws_bytes, cur.cuda_stream)
        check(rc, "pvn3d_icp_refine_batch" + ("" if self.cluster_bw is None else "_clustered"))
        return self.poses[:b], self.iters[:b], self.err[:b], self.refined[:b]


_INT32_LIMIT = 1 << 31


def _check_dev(t: torch.Tensor, dt, dev, what: str) -> None:
    if not (t.is_cuda and t.is_contiguous() and t.dtype == dt and (dev is None or t.device == dev)):
        raise ValueError(f"{what}: expected a contiguous {dt} CUDA tensor" + ("" if dev is None else f" on {dev}"))


def depth_to_cloud(depth: torch.Tensor, K: torch.Tensor, cam_scale: torch.Tensor, *, out=None):
    """Basic_Utils.dpt_2_cld (lib/utils/basic_utils.py:381-399) for every pixel of a batch, on device.
    depth [B,H,W] f32 (convert a uint16 depth PNG with .float(), as the reference's .astype(np.float32)),
    K [B,3,3] f32 (per frame), cam_scale [B] f32.  Returns (cloud [B,H*W,3] f32, valid [B,H*W] u8) in
    raster order: valid = depth > 1e-6; pt2 = depth / cam_scale, pt0 = (col - cx) * pt2 / fx,
    pt1 = (row - cy) * pt2 / fy in float32; invalid pixels hold (0, 0, 0).  `out` = (cloud, valid)
    to write into.  Runs on the current stream, no host sync."""
    if depth.dim() != 3 or K.shape != (depth.size(0), 3, 3) or cam_scale.shape != (depth.size(0),):
        raise ValueError(f"depth_to_cloud: expected depth [B,H,W], K [B,3,3], cam_scale [B]; got "
                         f"{tuple(depth.shape)}, {tuple(K.shape)}, {tuple(cam_scale.shape)}")
    dev = depth.device
    for t, name in ((depth, "depth"), (K, "K"), (cam_scale, "cam_scale")):
        _check_dev(t, torch.float32, dev, f"depth_to_cloud: {name}")
    b, h, w = depth.shape
    if b * h * w >= _INT32_LIMIT:
        raise ValueError(f"depth_to_cloud: B*H*W = {b * h * w} pixels needs 64-bit indexing")
    if out is None:
        cloud = torch.empty((b, h * w, 3), dtype=torch.float32, device=dev)
        valid = torch.empty((b, h * w), dtype=torch.uint8, device=dev)
    else:
        cloud, valid = out
        if cloud.shape != (b, h * w, 3) or valid.shape != (b, h * w):
            raise ValueError("depth_to_cloud: `out` shapes do not match the depth batch")
        _check_dev(cloud, torch.float32, dev, "depth_to_cloud: out cloud")
        _check_dev(valid, torch.uint8, dev, "depth_to_cloud: out valid")
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.pvn3d_depth_to_cloud(ptr(depth), ptr(K), ptr(cam_scale), b, h, w, ptr(cloud), ptr(valid),
                                      torch.cuda.current_stream(dev).cuda_stream)
    check(rc, "pvn3d_depth_to_cloud")
    return cloud, valid


def fill_label(cloud: torch.Tensor, valid: torch.Tensor, pcld: torch.Tensor, point_labels: torch.Tensor, *,
               out=None, nn_idx=None) -> torch.Tensor:
    """pvn3d/eval_icp.py:388-422 (fill_label_item) on device: every valid pixel of cloud [B,P,3] f32 /
    valid [B,P] u8 takes point_labels[b, j] [B,N] i32 of its nearest sampled point j of pcld [B,N,3] f32
    -- float64 distance (dx*dx + dy*dy) + dz*dz, lowest j on exact ties, which is sklearn
    NearestNeighbors(n_neighbors=1)'s answer wherever the two best distances differ.  Invalid pixels
    get 0.  Returns labels [B,P] i32 (`out` if given); `nn_idx` [B,P] i32, if given, receives j (-1 for
    invalid pixels).  Runs on the current stream, no host sync."""
    if cloud.dim() != 3 or cloud.size(2) != 3 or pcld.dim() != 3 or pcld.size(2) != 3:
        raise ValueError(f"fill_label: expected cloud [B,P,3] and pcld [B,N,3]; got {tuple(cloud.shape)}, "
                         f"{tuple(pcld.shape)}")
    b, p = cloud.shape[:2]
    n = pcld.size(1)
    if valid.shape != (b, p) or pcld.size(0) != b or point_labels.shape != (b, n) or n < 1 or p < 1:
        raise ValueError(f"fill_label: shapes do not agree: cloud {tuple(cloud.shape)}, valid {tuple(valid.shape)}, "
                         f"pcld {tuple(pcld.shape)}, point_labels {tuple(point_labels.shape)}")
    dev = cloud.device
    for t, dt, name in ((cloud, torch.float32, "cloud"), (valid, torch.uint8, "valid"), (pcld, torch.float32, "pcld"),
                        (point_labels, torch.int32, "point_labels")):
        _check_dev(t, dt, dev, f"fill_label: {name}")
    lib = _lib.load()
    ws_bytes = int(lib.pvn3d_label_fill_workspace_bytes(b, n))
    if ws_bytes == 0 or b * p >= _INT32_LIMIT:
        raise ValueError(f"fill_label: B={b}, P={p}, N={n} needs 64-bit indexing")
    labels = torch.empty((b, p), dtype=torch.int32, device=dev) if out is None else out
    for t, name in ((labels, "out"), (nn_idx, "nn_idx")):
        if t is not None:
            if t.shape != (b, p):
                raise ValueError(f"fill_label: {name} must be [B,P]")
            _check_dev(t, torch.int32, dev, f"fill_label: {name}")
    ws, ws_ptr = _aligned(ws_bytes, dev)
    with torch.cuda.device(dev):
        rc = lib.pvn3d_label_fill(ptr(cloud), ptr(valid), p, ptr(pcld), ptr(point_labels), b, n, ptr(labels),
                                  ptr(nn_idx), ws_ptr, ws_bytes, torch.cuda.current_stream(dev).cuda_stream)
    check(rc, "pvn3d_label_fill")
    return labels


def dpt_2_cld(dpt, cam_scale, K, device="cuda"):
    """lib/utils/basic_utils.py:381-399 for one frame, computed on the GPU: dpt [H,W] (or [H,W,C]: channel
    0), cam_scale and K [3,3] -> (cld [n,3] float32, choose [n] uint32) over the n pixels with dpt > 1e-6,
    in raster order; (None, None) when there is none.  dpt, K and cam_scale are taken as float32: the
    reference's arithmetic for float32 K (eval_icp's cam_scale is float32), and for any K under NumPy 1.x."""
    dev = _cuda_device(device, "dpt_2_cld (pvn3d_b200)")
    d = dpt.detach().cpu().numpy() if torch.is_tensor(dpt) else np.asarray(dpt)
    if d.ndim > 2:
        d = d[:, :, 0]
    if d.ndim != 2:
        raise ValueError(f"dpt_2_cld: expected an [H,W] depth image, got shape {d.shape}")
    k = K.detach().cpu().numpy() if torch.is_tensor(K) else np.asarray(K)
    k = np.ascontiguousarray(k, np.float32).reshape(1, 3, 3)
    h, w = d.shape
    td = torch.from_numpy(np.ascontiguousarray(d, np.float32)).reshape(1, h, w).to(dev)
    cs = torch.tensor([float(np.float32(cam_scale))], dtype=torch.float32).to(dev)
    cloud, valid = depth_to_cloud(td, torch.from_numpy(k).to(dev), cs)
    v = valid[0].cpu().numpy().astype(bool)
    choose = np.nonzero(v)[0].astype(np.uint32)
    if len(choose) < 1:
        return None, None
    return cloud[0].cpu().numpy()[v], choose


class DepthIcpRefiner:
    """eval_icp's refinement (pvn3d/eval_icp.py:224-291, label_type='predmsk') on full-resolution depth,
    batched and sync-free: back-project every pixel (depth_to_cloud), give each valid pixel a label
    (fill_label from the network's sampled cloud, or a given label image), then run IcpRefiner with
    n_pts = H*W on the pixel cloud -- invalid pixels carry class 0 and are never selected.  So each
    object's scene set is its pixels in raster order: max_pts of them by the stride
    floor(j*cnt/max_pts), skipped below min_pts, the biggest flat mean-shift cluster, then my_icp.

    Defaults are eval_icp's: max_pts=2000 (n_sample_points), min_pts=1500, cluster_bandwidth=0.06,
    max_iter=500, tol=1e-9.  Deliberate differences from the reference, shared with IcpRefiner: the
    stride replaces np.random.shuffle's subset, and a class the solver did not find passes its pose
    through (the reference runs ICP from a zero pose)."""

    def __init__(self, models, n_cls: int, batch: int, height: int = 480, width: int = 640, *, max_pts: int = 2000,
                 min_pts: int = 1500, cluster_bandwidth=0.06, max_iter: int = 500, tol: float = 1e-9,
                 cluster_max_iter: int = 300, device="cuda"):
        self.dev = _cuda_device(device, "DepthIcpRefiner")
        self.h, self.w, self.b = int(height), int(width), int(batch)
        if self.h < 1 or self.w < 1 or self.b < 1:
            raise ValueError(f"batch={batch}, height={height}, width={width}: all must be >= 1")
        if self.b * self.h * self.w >= _INT32_LIMIT:
            raise ValueError(f"DepthIcpRefiner: {self.b}x{self.h}x{self.w} pixels needs 64-bit indexing")
        hw = self.h * self.w
        self.icp = IcpRefiner(models, n_cls, self.b, hw, max_pts=max_pts, min_pts=min_pts, max_iter=max_iter, tol=tol,
                              cluster_bandwidth=cluster_bandwidth, cluster_max_iter=cluster_max_iter, device=self.dev)
        self.n_cls = self.icp.n_cls
        #: the pixel cloud [B,H*W,3] f32, its validity [B,H*W] u8 and per-pixel labels [B,H*W] i32 (0 where
        #: invalid) of the last refine(): refiner-owned, valid until the next refine() on the same stream
        self.cloud = torch.empty((self.b, hw, 3), dtype=torch.float32, device=self.dev)
        self.valid = torch.empty((self.b, hw), dtype=torch.uint8, device=self.dev)
        self.labels = torch.empty((self.b, hw), dtype=torch.int32, device=self.dev)

    @property
    def cluster_pts(self):
        """[B,n_cls] i32: pixels each fit of the last refine() used after the cluster filter (0 when skipped)"""
        return self.icp.cluster_pts

    def kept_points(self) -> torch.Tensor:
        """IcpRefiner.kept_points over the pixel cloud: the fits' pixel indices (row-major y*W + x)"""
        return self.icp.kept_points()

    def refine(self, depth: torch.Tensor, K: torch.Tensor, cam_scale: torch.Tensor, poses: torch.Tensor,
               present: torch.Tensor, *, pcld: torch.Tensor = None, point_labels: torch.Tensor = None,
               label_image: torch.Tensor = None):
        """depth [B,H,W] f32, K [B,3,3] f32, cam_scale [B] f32, poses [B,n_cls,3,4] f32 and present
        [B,n_cls] u8 (FramePoseSolver.solve()), and the labels as either
          pcld [B,N,3] f32 + point_labels [B,N] i32: the network's sampled cloud and its labels (the
            solver's new_mask, or seg_argmax), filled to every pixel (eval_icp's fill_label_item); or
          label_image [B,H,W] integer: a label per pixel (eval_icp's eval_item, the ground-truth mask).
        Returns IcpRefiner.refine's (poses f64, iters, err, refined), views of refiner-owned buffers.
        Everything runs on the current stream; no host sync."""
        b = depth.size(0) if depth.dim() == 3 else -1
        if not (1 <= b <= self.b and depth.shape[1:] == (self.h, self.w)):
            raise ValueError(f"DepthIcpRefiner.refine: depth must be [B<={self.b},{self.h},{self.w}], "
                             f"got {tuple(depth.shape)}")
        if (label_image is None) == (pcld is None and point_labels is None):
            raise ValueError("DepthIcpRefiner.refine: pass either pcld and point_labels, or label_image")
        if label_image is None and (pcld is None or point_labels is None):
            raise ValueError("DepthIcpRefiner.refine: pcld and point_labels go together")
        cloud, valid, labels = self.cloud[:b], self.valid[:b], self.labels[:b]
        with torch.cuda.device(self.dev):
            depth_to_cloud(depth, K, cam_scale, out=(cloud, valid))
            if label_image is None:
                fill_label(cloud, valid, pcld, point_labels, out=labels)
            else:
                if label_image.shape != (b, self.h, self.w) or label_image.device != self.dev:
                    raise ValueError(f"DepthIcpRefiner.refine: label_image must be [{b},{self.h},{self.w}] on "
                                     f"{self.dev}")
                torch.mul(label_image.reshape(b, -1), valid, out=labels)
            return self.icp.refine(cloud, labels, poses, present)


def my_icp(A, B, init_pose=None, max_iterations=20, tolerance=0.001, device="cuda"):
    """lib/utils/icp/icp.py:141-192: refine init_pose (4x4, rigid; None = identity) so that the model
    A [P,3] fits the scene points B [n,3].  A and B are used as float32 (as eval_icp produces them),
    init_pose as float64.  Returns (T 4x4 float64, distances [n] float64 of the last iteration,
    i = the last loop index).  CUDA only."""
    dev = _cuda_device(device, "my_icp (pvn3d_b200)")
    a, bq = _points(A, "A"), _points(B, "B")
    if len(a) == 0 or len(bq) == 0:
        raise ValueError("my_icp: A and B must be non-empty")
    if int(max_iterations) < 1:
        raise ValueError("my_icp: max_iterations must be >= 1 (the reference returns no distances otherwise)")
    if init_pose is None:
        init = np.eye(4)
    else:
        init = init_pose.detach().cpu().numpy() if torch.is_tensor(init_pose) else np.asarray(init_pose)
        init = np.asarray(init, np.float64)
        if init.shape != (4, 4) or not np.array_equal(init[3], [0.0, 0.0, 0.0, 1.0]):
            raise ValueError("my_icp: init_pose must be a 4x4 rigid transform (last row 0 0 0 1)")
    lib = _lib.load()
    models = IcpModels(a, np.array([0, len(a)], np.int32), dev)
    n = len(bq)
    ws_bytes = int(lib.pvn3d_icp_workspace_bytes(1, n, 1, n))
    ws, ws_ptr = _aligned(ws_bytes, dev)
    d_b = torch.from_numpy(bq).to(dev)
    d_init = torch.from_numpy(np.ascontiguousarray(init[:3])).to(dev)
    pose = torch.empty((3, 4), dtype=torch.float64, device=dev)
    dist = torch.empty((n,), dtype=torch.float64, device=dev)
    it = torch.empty((1,), dtype=torch.int32, device=dev)
    err = torch.empty((1,), dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        rc = lib.pvn3d_icp_fit(models.ptr, 0, ptr(d_b), n, ptr(d_init), int(max_iterations), float(tolerance),
                               ptr(pose), ptr(dist), ptr(it), ptr(err), ws_ptr, ws_bytes,
                               torch.cuda.current_stream(dev).cuda_stream)
    check(rc, "pvn3d_icp_fit")
    T = np.eye(4)
    T[:3] = pose.cpu().numpy()
    return T, dist.cpu().numpy(), int(it.cpu()[0])


def get_cld_bigest_clus(p3ds, radius: float = 0.06, device="cuda"):
    """pvn3d/eval_icp.py:56-64: p3ds[labels == 0] for the labels of sklearn's MeanShift(bandwidth=radius,
    bin_seeding=True) -- the biggest flat mean-shift cluster -- in input order.  p3ds [n,3], n <= 4096, is
    clustered as float64 on the GPU; the result keeps p3ds's type and dtype (an array or a tensor on its
    own device), as the reference's indexing does.  CUDA only."""
    from .meanshift import flat_mean_shift

    a = p3ds.detach().cpu().numpy() if torch.is_tensor(p3ds) else np.asarray(p3ds)
    _, labels, _ = flat_mean_shift(a, radius, device=device)
    keep = np.where(labels == 0)[0]
    if torch.is_tensor(p3ds):
        return p3ds[torch.from_numpy(keep).to(p3ds.device), :]
    return a[keep, :]
