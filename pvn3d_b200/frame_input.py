"""The network input of an RGB-D frame on the GPU -- what the datasets' get_item builds on the CPU
(pvn3d/datasets/ycb/ycb_dataset.py:185-233, pvn3d/datasets/linemod/linemod_dataset.py:211-271) -- by
csrc/normals.cu after icp.depth_to_cloud:

    fib = FrameInputBuilder(batch, n_points=12288, normals="full", device="cuda")
    cld_rgb_nrm, rgb, choose, pcld, ok = fib.build(depth, K, cam_scale, rgb, seed)
    kp, seg, ctr = FusedPVN3D(model).forward(cld_rgb_nrm, rgb, choose)
    nrm = estimate_normals(cld)                  # get_normal for one cloud: [n,4] (normal, curvature)

Deliberate differences from get_item, all documented in INTEGRATION.md section 2a:
  * the subset is the N valid pixels with the smallest seeded 64-bit keys (pvn3d_frame_sample in
    include/pvn3d_b200.h), not np.random.shuffle's: the same distribution, reproducible from the seed;
  * normals are the mathematically defined ones of the exact 50-neighbour covariance in float64, not
    PCL's float32 rounding; a neighbourhood of 50 coincident points gets (0, 0, 0), which is what
    get_item's `normal[np.isnan(normal)] = 0.0` makes of PCL's NaN there;
  * a frame with fewer than 400 valid pixels is not dropped (get_item returns None) but flagged ok = 0
    and zero-filled, so the batch keeps its shape;
  * depth is taken as given unless fill="multiscale", which runs Basic_Utils.fill_missing (YCB's
    get_item fills every frame) on the GPU first (depth_fill.DepthFiller).
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from ._lib import check, ptr
from .depth_fill import DepthFiller
from .icp import _INT32_LIMIT, _aligned, _check_dev, _cuda_device, depth_to_cloud

K_SEARCH = 50        #: neighbours per normal (the reference's ne.set_KSearch(50))
MIN_VALID = 400      #: get_item returns None below this many valid pixels
NORMAL_MODES = ("full", "sampled")
FILL_MODES = (None, "multiscale")


def _knn_normals(lib, ref, ref_valid, query, frame_ok, normals_out, row_stride, *, curv=None, normals64=None,
                 nn_idx=None, ws=None):
    """pvn3d_knn_normals on the current stream: ref [B,R,3] f32 (+ ref_valid [B,R] u8 or None), query [B,Q,3]
    f32 -> normals_out rows of `row_stride` floats.  ws = (owner, address, bytes) or None to allocate."""
    b, r = ref.shape[:2]
    q = query.size(1)
    if ws is None:
        nbytes = int(lib.pvn3d_knn_normals_workspace_bytes(b, r, q))
        if nbytes == 0:
            raise ValueError(f"knn normals: B={b}, R={r}, Q={q} needs 64-bit indexing")
        ws = _aligned(nbytes, ref.device) + (nbytes,)
    dev = ref.device
    with torch.cuda.device(dev):
        rc = lib.pvn3d_knn_normals(ptr(ref), ptr(ref_valid), r, ptr(query), q, b, ptr(frame_ok), ptr(normals_out),
                                   int(row_stride), ptr(curv), ptr(normals64), ptr(nn_idx), ws[1], ws[2],
                                   torch.cuda.current_stream(dev).cuda_stream)
    check(rc, "pvn3d_knn_normals")


class FrameInputBuilder:
    """Batched, sync-free construction of PVN3D's input (cld_rgb_nrm, rgb, choose) from depth + RGB.

    normals  "full": each sampled point's 50 neighbours are searched among every valid pixel of its frame,
               as ycb_dataset.py:210-212 estimates normals on the whole cloud before sampling (only the kept
               points' normals are computed: the values are the same);
             "sampled": among the frame's N sampled points, wrap duplicates included, as
               linemod_dataset.py:269-270 does.
    fill     None: build() takes depth as given; "multiscale": build() first fills it as YCB's get_item does
             (Basic_Utils.fill_missing(dpt, cam_scale, 1), ycb_dataset.py:206) into `filled` [B,H,W] f32 and
             back-projects that.
    debug    keep the neighbour indices [B,N,50] i32 (`nn_idx`: pixel indices in "full" mode, sample
             indices in "sampled" mode), the float64 normals [B,N,3] (`normals64`) and the curvature
             [B,N] f32 (`curvature`) of the last build().
    """

    def __init__(self, batch: int, n_points: int = 12288, height: int = 480, width: int = 640, *,
                 normals: str = "full", fill: str = None, debug: bool = False, device="cuda"):
        self.dev = _cuda_device(device, "FrameInputBuilder")
        self.b, self.n, self.h, self.w = int(batch), int(n_points), int(height), int(width)
        if normals not in NORMAL_MODES:
            raise ValueError(f"normals={normals!r}: one of {NORMAL_MODES}")
        self.mode = normals
        if fill not in FILL_MODES:
            raise ValueError(f"fill={fill!r}: one of {FILL_MODES}")
        if self.b < 1 or self.h < 1 or self.w < 1:
            raise ValueError(f"batch={batch}, height={height}, width={width}: all must be >= 1")
        if self.n < K_SEARCH:
            raise ValueError(f"n_points={n_points}: at least {K_SEARCH} (the normals' neighbourhood)")
        hw = self.h * self.w
        self.lib = _lib.load()
        n_ref = hw if normals == "full" else self.n
        self._ws_s_bytes = int(self.lib.pvn3d_frame_sample_workspace_bytes(self.b, hw, self.n))
        self._ws_n_bytes = int(self.lib.pvn3d_knn_normals_workspace_bytes(self.b, n_ref, self.n))
        if self._ws_s_bytes == 0 or self._ws_n_bytes == 0 or self.b * hw >= _INT32_LIMIT:
            raise ValueError(f"FrameInputBuilder: {self.b}x{self.h}x{self.w} pixels / {self.n} points needs "
                             "64-bit indexing")
        self._ws_s = _aligned(self._ws_s_bytes, self.dev) + (self._ws_s_bytes,)
        self._ws_n = _aligned(self._ws_n_bytes, self.dev) + (self._ws_n_bytes,)
        f32 = dict(dtype=torch.float32, device=self.dev)
        #: the back-projected pixels [B,H*W,3] f32 and their validity [B,H*W] u8 of the last build()
        self.cloud = torch.empty((self.b, hw, 3), **f32)
        self.valid = torch.empty((self.b, hw), dtype=torch.uint8, device=self.dev)
        self.cld_rgb_nrm = torch.empty((self.b, self.n, 9), **f32)
        self.rgb = torch.empty((self.b, 3, self.h, self.w), **f32)
        self.choose = torch.empty((self.b, 1, self.n), dtype=torch.int64, device=self.dev)
        self.pcld = torch.empty((self.b, self.n, 3), **f32)
        self.ok = torch.empty((self.b,), dtype=torch.uint8, device=self.dev)
        self.labels = torch.empty((self.b, self.n), dtype=torch.int32, device=self.dev)
        self.filler = self.filled = None
        if fill == "multiscale":
            self.filler = DepthFiller(self.b, self.h, self.w, device=self.dev)
            #: the filled depth [B,H,W] f32 of the last build()
            self.filled = self.filler.out
        self.nn_idx = self.normals64 = self.curvature = None
        if debug:
            self.nn_idx = torch.empty((self.b, self.n, K_SEARCH), dtype=torch.int32, device=self.dev)
            self.normals64 = torch.empty((self.b, self.n, 3), dtype=torch.float64, device=self.dev)
            self.curvature = torch.empty((self.b, self.n), **f32)

    def build(self, depth: torch.Tensor, K: torch.Tensor, cam_scale: torch.Tensor, rgb: torch.Tensor, seed: int, *,
              label_image: torch.Tensor = None):
        """depth [B,H,W] f32 (filled first when the builder was made with fill="multiscale"), K [B,3,3] f32, cam_scale [B] f32, rgb
        [B,3,H,W] uint8 or float32 (the CHW image the network takes: BGR for LineMOD, RGB for YCB), seed a
        non-negative int (the subset is a function of seed, frame index and pixel index).

        Returns (cld_rgb_nrm [B,N,9] f32, rgb [B,3,H,W] f32, choose [B,1,N] i64, pcld [B,N,3] f32, ok [B] u8),
        and labels [B,N] i32 = label_image[b].flatten()[choose] as a sixth element when label_image [B,H,W]
        (integer) is given.  Frames with ok = 0 (fewer than 400 valid pixels) are zero.  The tensors are views
        of builder-owned buffers, valid until the next build() on the same stream.  Everything runs on the
        current stream; no host sync."""
        b = depth.size(0) if depth.dim() == 3 else -1
        if not (1 <= b <= self.b and depth.shape[1:] == (self.h, self.w)):
            raise ValueError(f"FrameInputBuilder.build: depth must be [B<={self.b},{self.h},{self.w}], "
                             f"got {tuple(depth.shape)}")
        if rgb.shape != (b, 3, self.h, self.w) or rgb.dtype not in (torch.uint8, torch.float32):
            raise ValueError(f"FrameInputBuilder.build: rgb must be [{b},3,{self.h},{self.w}] uint8 or float32, got "
                             f"{tuple(rgb.shape)} {rgb.dtype}")
        _check_dev(rgb, rgb.dtype, self.dev, "FrameInputBuilder.build: rgb")
        seed = int(seed)
        if not 0 <= seed < 1 << 64:
            raise ValueError(f"FrameInputBuilder.build: seed={seed} must be in [0, 2**64)")
        lab = None
        if label_image is not None:
            if label_image.shape != (b, self.h, self.w) or label_image.device != self.dev:
                raise ValueError(f"FrameInputBuilder.build: label_image must be [{b},{self.h},{self.w}] on {self.dev}")
            lab = label_image.reshape(b, -1).to(torch.int32).contiguous()
        hw = self.h * self.w
        cloud, valid, ok = self.cloud[:b], self.valid[:b], self.ok[:b]
        cld, pcld, choose, labels = self.cld_rgb_nrm[:b], self.pcld[:b], self.choose[:b], self.labels[:b]
        with torch.cuda.device(self.dev):
            if self.filler is not None:
                depth = self.filler.fill(depth, cam_scale)
            depth_to_cloud(depth, K, cam_scale, out=(cloud, valid))
            rc = self.lib.pvn3d_frame_sample(
                ptr(cloud), ptr(valid), ptr(rgb), int(rgb.dtype == torch.uint8), ptr(lab), b, hw, self.n, seed,
                ptr(cld), 9, ptr(pcld), ptr(choose), ptr(labels) if lab is not None else 0, ptr(ok),
                self._ws_s[1], self._ws_s[2], torch.cuda.current_stream(self.dev).cuda_stream)
            check(rc, "pvn3d_frame_sample")
            if self.mode == "full":
                ref, ref_valid = cloud, valid
            else:
                ref, ref_valid = pcld, None
            dbg = {}
            if self.nn_idx is not None:
                dbg = dict(curv=self.curvature[:b], normals64=self.normals64[:b], nn_idx=self.nn_idx[:b])
            _knn_normals(self.lib, ref, ref_valid, pcld, ok, cld[:, :, 6:], 9, ws=self._ws_n, **dbg)
            self.rgb[:b].copy_(rgb)
            if lab is not None:
                lab.record_stream(torch.cuda.current_stream(self.dev))
        out = (cld, self.rgb[:b], choose, pcld, ok)
        return out + (labels,) if lab is not None else out


def estimate_normals(cld, k: int = K_SEARCH, device="cuda") -> np.ndarray:
    """get_normal (ycb_dataset.py:147-157, linemod_dataset.py:152-162) for one cloud, on the GPU: cld [n,3]
    (taken as float32) -> [n,4] float32 (normal_x, normal_y, normal_z, curvature), the layout of PCL's
    NormalEstimation(...).compute().to_array().  Neighbours: the exact 50 nearest points of the cloud (the
    point itself included); the normal is the smallest-eigenvalue eigenvector of their covariance, turned
    towards the origin; curvature = lambda0 / trace.  Where PCL would return NaN (coincident neighbours),
    or for a non-finite point, the row is zero; a cloud of fewer than 50 finite points has zero rows only."""
    if int(k) != K_SEARCH:
        raise ValueError(f"estimate_normals: k={k}; the kernel searches exactly {K_SEARCH} neighbours")
    dev = _cuda_device(device, "estimate_normals")
    a = cld.detach().cpu().numpy() if torch.is_tensor(cld) else np.asarray(cld)
    a = np.ascontiguousarray(a, np.float32)
    if a.ndim != 2 or a.shape[1] != 3 or len(a) < 1:
        raise ValueError(f"estimate_normals: expected a non-empty [n,3] cloud, got shape {a.shape}")
    n = len(a)
    pts = torch.from_numpy(a).to(dev).view(1, n, 3)
    out = torch.empty((1, n, 4), dtype=torch.float32, device=dev)
    curv = torch.empty((1, n), dtype=torch.float32, device=dev)
    _knn_normals(_lib.load(), pts, None, pts, None, out, 4, curv=curv)
    out[0, :, 3] = curv[0]
    return out[0].cpu().numpy()
