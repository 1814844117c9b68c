"""YCB's depth completion on the GPU: Basic_Utils.fill_missing (lib/utils/basic_utils.py:436-456), which
ycb_dataset.py:206 runs on every frame before dpt_2_cld -- ip_basic's fill_in_multiscale with max_depth 3,
no extrapolation and the bilateral blur -- by csrc/depth_fill.cu:

    filler = DepthFiller(batch, 480, 640, device="cuda")
    filled = filler.fill(depth, cam_scale)           # depth [B,H,W] f32 raw units, cam_scale [B] f32
    dpt = fill_missing(dpt, cam_scale, 1)            # the one-frame numpy drop-in

Steps 1-9 (everything before the bilateral) are bit-exact; the bilateral is cv2's float32 algorithm with
float32 sums, within 3 * 2^-20 * max(|min|, |max|) of the pre-bilateral image (include/pvn3d_b200.h).
Only fill_type 'multiscale' with extrapolate False and blur_type 'bilateral' -- the arguments fill_missing is
called with -- is implemented; anything else raises.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from ._lib import check, ptr
from .icp import _aligned, _check_dev, _cuda_device


class DepthFiller:
    """Batched, sync-free fill_missing for frames of one size.  Owns its workspace and output.

    debug  keep `stages` [B,4,H,W] f32 (s4, s5, the bilateral's input, the bilateral's output, before the
           inversion) and `top_rows` [B,2,W] i32 (top1, top2) of the last fill().
    """

    def __init__(self, batch: int, height: int = 480, width: int = 640, *, debug: bool = False, device="cuda"):
        self.dev = _cuda_device(device, "DepthFiller")
        self.b, self.h, self.w = int(batch), int(height), int(width)
        if self.b < 1 or self.h < 1 or self.w < 1:
            raise ValueError(f"batch={batch}, height={height}, width={width}: all must be >= 1")
        self.lib = _lib.load()
        self._ws_bytes = int(self.lib.pvn3d_depth_fill_workspace_bytes(self.b, self.h, self.w))
        if self._ws_bytes == 0:
            raise ValueError(f"DepthFiller: {self.b}x{self.h}x{self.w} pixels needs 64-bit indexing")
        self._ws = _aligned(self._ws_bytes, self.dev)
        self.out = torch.empty((self.b, self.h, self.w), dtype=torch.float32, device=self.dev)
        self.stages = self.top_rows = None
        if debug:
            self.stages = torch.empty((self.b, 4, self.h, self.w), dtype=torch.float32, device=self.dev)
            self.top_rows = torch.empty((self.b, 2, self.w), dtype=torch.int32, device=self.dev)

    def fill(self, depth: torch.Tensor, cam_scale: torch.Tensor, scale_2_80m: float = 1.0, out=None) -> torch.Tensor:
        """depth [B<=batch,H,W] f32 (raw units, as the depth PNG holds them), cam_scale [B] f32 ->
        the filled depth [B,H,W] f32 in the same units, into `out` when given, else a view of the
        filler's buffer (valid until the next fill() on the same stream).  Current stream; no host sync."""
        b = depth.size(0) if depth.dim() == 3 else -1
        if not (1 <= b <= self.b and depth.shape[1:] == (self.h, self.w)):
            raise ValueError(f"DepthFiller.fill: depth must be [B<={self.b},{self.h},{self.w}], got {tuple(depth.shape)}")
        _check_dev(depth, torch.float32, self.dev, "DepthFiller.fill: depth")
        if cam_scale.shape != (b,):
            raise ValueError(f"DepthFiller.fill: cam_scale must be [{b}], got {tuple(cam_scale.shape)}")
        _check_dev(cam_scale, torch.float32, self.dev, "DepthFiller.fill: cam_scale")
        s2s = float(np.float32(scale_2_80m))
        if not (np.isfinite(s2s) and s2s > 0):
            raise ValueError(f"DepthFiller.fill: scale_2_80m={scale_2_80m} must be finite and > 0")
        if out is None:
            out = self.out[:b]
        elif out.shape != (b, self.h, self.w):
            raise ValueError(f"DepthFiller.fill: out must be [{b},{self.h},{self.w}], got {tuple(out.shape)}")
        _check_dev(out, torch.float32, self.dev, "DepthFiller.fill: out")
        stages = None if self.stages is None else self.stages[:b]
        tops = None if self.top_rows is None else self.top_rows[:b]
        with torch.cuda.device(self.dev):
            rc = self.lib.pvn3d_depth_fill(ptr(depth), ptr(cam_scale), s2s, b, self.h, self.w, ptr(out), ptr(stages),
                                           ptr(tops), self._ws[1], self._ws_bytes,
                                           torch.cuda.current_stream(self.dev).cuda_stream)
        check(rc, "pvn3d_depth_fill")
        return out


_FILLERS: dict = {}


def fill_missing(dpt, cam_scale, scale_2_80m=1.0, fill_type: str = "multiscale", extrapolate: bool = False,
                 blur_type: str = "bilateral", device="cuda") -> np.ndarray:
    """Basic_Utils.fill_missing for one frame on the GPU: dpt [H,W] (any real dtype, taken as float32, raw
    units) -> [H,W] float32.  Only the arguments the datasets use are implemented: fill_type 'multiscale',
    extrapolate False, blur_type 'bilateral'; fill_in_fast, extrapolation and the Gaussian blur raise
    ValueError."""
    if fill_type != "multiscale":
        raise ValueError(f"fill_missing: fill_type={fill_type!r}; only 'multiscale' is implemented")
    if extrapolate:
        raise ValueError("fill_missing: extrapolate=True is not implemented")
    if blur_type != "bilateral":
        raise ValueError(f"fill_missing: blur_type={blur_type!r}; only 'bilateral' is implemented")
    a = dpt.detach().cpu().numpy() if torch.is_tensor(dpt) else np.asarray(dpt)
    if a.ndim != 2 or a.size == 0:
        raise ValueError(f"fill_missing: expected a non-empty [H,W] depth image, got shape {a.shape}")
    dev = _cuda_device(device, "fill_missing")
    key = (dev, a.shape)
    filler = _FILLERS.get(key)
    if filler is None:
        filler = _FILLERS[key] = DepthFiller(1, a.shape[0], a.shape[1], device=dev)
    d = torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)[None]
    cs = torch.tensor([float(np.float32(cam_scale))], dtype=torch.float32, device=dev)
    return filler.fill(d, cs, scale_2_80m)[0].cpu().numpy()
