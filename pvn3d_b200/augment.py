"""get_item's training augmentation on the GPU: ColorJitter(0.2, 0.2, 0.2, 0.05), rgb_add_noise and add_real_back
(ycb_dataset.py:84-177,191-204, linemod_dataset.py:103-188,211-240) for a batch of decoded frames, by
csrc/augment.cu:

    aug = FrameAugmenter(batch, "ycb", 480, 640, device="cuda")
    params = aug.draw(seed, kinds)                         # kinds [B]: YCB 0 real / 1 syn;
                                                           #   LineMOD 0 real png / 1 render / 2 fuse
    rgb_chw, depth = aug.apply(rgb, depth, labels, back_rgb, back_labels, back_depth, params)

The draw turns (seed, frame, kind) into one parameter record per frame with the reference's decision structure and
distributions (Philox4x32-10; not numpy's or torch's streams).  The apply runs every operation in the precision
of the library the reference calls: the colour conversions, the Gaussian blur and the composite are bit-exact to
cv2 4.13 / PIL 12.2, filter2D is within 1 of cv2 (include/pvn3d_b200.h).  The frame's kind and its background
frame (real_gen) are the caller's choice, as in the reference.  The outputs feed FrameInputBuilder.build /
train_batch(fill="multiscale") directly: rgb [B,3,H,W] uint8 in the network's channel order (YCB RGB, LineMOD BGR)
and the composited depth [B,H,W] float32.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _lib
from ._lib import check, ptr
from .icp import _aligned, _check_dev, _cuda_device

DATASETS = {"ycb": 0, "linemod": 1}
#: frame kinds each dataset accepts
KINDS = {"ycb": {"real": 0, "syn": 1}, "linemod": {"real": 0, "render": 1, "fuse": 2}}
PARAMS_BYTES = 208          # sizeof(pvn3d_augment_params_t)
N_STAGES = 12


class FrameAugmenter:
    """Batched, sync-free training augmentation of frames of one size.  Owns its workspace and outputs.

    debug  keep `stages` [B,12,H,W,3] uint8 (after the jitter and flip; the first noise pass's hsv, sharpen,
           motion, gauss, noise; the composite; the second pass's five) and `noise` [B,2,2,H,W,3] float32 (per
           pass the noise and extra standard-normal fields) of the last apply().
    """

    def __init__(self, batch: int, dataset: str = "ycb", height: int = 480, width: int = 640, *, debug: bool = False,
                 device="cuda"):
        if dataset not in DATASETS:
            raise ValueError(f"FrameAugmenter: dataset={dataset!r}; one of {sorted(DATASETS)}")
        self.dev = _cuda_device(device, "FrameAugmenter")
        self.dataset = dataset
        self.b, self.h, self.w = int(batch), int(height), int(width)
        if self.b < 1 or self.h < 1 or self.w < 1:
            raise ValueError(f"batch={batch}, height={height}, width={width}: all must be >= 1")
        self.lib = _lib.load()
        self._ws_bytes = int(self.lib.pvn3d_augment_workspace_bytes(self.b, self.h, self.w))
        if self._ws_bytes == 0:
            raise ValueError(f"FrameAugmenter: {self.b}x{self.h}x{self.w}x3 bytes needs 64-bit indexing")
        self._ws = _aligned(self._ws_bytes, self.dev)
        self.params = torch.empty((self.b, PARAMS_BYTES), dtype=torch.uint8, device=self.dev)
        self.rgb_out = torch.empty((self.b, 3, self.h, self.w), dtype=torch.uint8, device=self.dev)
        self.depth_out = torch.empty((self.b, self.h, self.w), dtype=torch.float32, device=self.dev)
        self.stages = self.noise = None
        if debug:
            self.stages = torch.zeros((self.b, N_STAGES, self.h, self.w, 3), dtype=torch.uint8, device=self.dev)
            self.noise = torch.zeros((self.b, 2, 2, self.h, self.w, 3), dtype=torch.float32, device=self.dev)

    def _stream(self):
        return torch.cuda.current_stream(self.dev).cuda_stream

    def draw(self, seed: int, kinds) -> torch.Tensor:
        """kinds [B<=batch] (ints, or the names of KINDS[dataset]; a host sequence or a device int32 tensor) ->
        the records [B,208] uint8 on the device (pvn3d_augment_params_t; `records()` reads them on the host), a
        view of the augmenter's buffer valid until the next draw().  Current stream; no host sync for a device
        `kinds`."""
        if torch.is_tensor(kinds):
            k = kinds
            _check_dev(k, torch.int32, self.dev, "FrameAugmenter.draw: kinds")
        else:
            names = KINDS[self.dataset]
            vals = [names[x] if isinstance(x, str) else int(x) for x in kinds]
            if any(v not in names.values() for v in vals):
                raise ValueError(f"FrameAugmenter.draw: kinds must be in {names}, got {list(kinds)}")
            k = torch.tensor(vals, dtype=torch.int32).to(self.dev, non_blocking=True)
        b = k.numel()
        if not (k.dim() == 1 and 1 <= b <= self.b):
            raise ValueError(f"FrameAugmenter.draw: kinds must be [B<={self.b}], got {tuple(k.shape)}")
        out = self.params[:b]
        with torch.cuda.device(self.dev):
            rc = self.lib.pvn3d_augment_draw(ctypes.c_ulonglong(int(seed) & (2**64 - 1)), ptr(k), b,
                                             DATASETS[self.dataset], ptr(out), self._stream())
        check(rc, "pvn3d_augment_draw")
        return out

    def apply(self, rgb, depth, labels, back_rgb, back_labels, back_depth, params):
        """rgb [B,H,W,3] uint8 RGB as decoded, depth [B,H,W] float32 (raw units), labels [B,H,W] uint8 (or
        [B,H,W,3]: channel 0, as get_item takes it; 0 = background), the background frame back_rgb [B,H,W,3] uint8
        RGB, back_labels [B,H,W] or [B,H,W,3] uint8 and back_depth [B,H,W] float32, params [B,208] uint8 (draw() or
        `from_records`) -> (rgb [B,3,H,W] uint8, depth [B,H,W] float32), views of the augmenter's buffers valid
        until the next apply().  Frames without a background composite still need (any) background tensors of the
        right shape.  Current stream; no host sync."""
        b = rgb.size(0) if rgb.dim() == 4 else -1
        hw = (self.h, self.w)
        if not (1 <= b <= self.b and rgb.shape[1:] == (*hw, 3)):
            raise ValueError(f"FrameAugmenter.apply: rgb must be [B<={self.b},{self.h},{self.w},3], got "
                             f"{tuple(rgb.shape)}")
        if labels.dim() == 4 and labels.shape[-1] == 3:
            labels = labels[..., 0].contiguous()
        for name, t, dt, shape in (("rgb", rgb, torch.uint8, (b, *hw, 3)), ("depth", depth, torch.float32, (b, *hw)),
                                   ("labels", labels, torch.uint8, (b, *hw)),
                                   ("back_rgb", back_rgb, torch.uint8, (b, *hw, 3)),
                                   ("back_depth", back_depth, torch.float32, (b, *hw)),
                                   ("params", params, torch.uint8, (b, PARAMS_BYTES))):
            if tuple(t.shape) != shape:
                raise ValueError(f"FrameAugmenter.apply: {name} must be {list(shape)}, got {tuple(t.shape)}")
            _check_dev(t, dt, self.dev, f"FrameAugmenter.apply: {name}")
        if back_labels.shape == (b, *hw):
            ch = 1
        elif back_labels.shape == (b, *hw, 3):
            ch = 3
        else:
            raise ValueError(f"FrameAugmenter.apply: back_labels must be [{b},{self.h},{self.w}] or [..., 3], got "
                             f"{tuple(back_labels.shape)}")
        _check_dev(back_labels, torch.uint8, self.dev, "FrameAugmenter.apply: back_labels")
        rgb_out, depth_out = self.rgb_out[:b], self.depth_out[:b]
        stages = None if self.stages is None else self.stages[:b]
        noise = None if self.noise is None else self.noise[:b]
        with torch.cuda.device(self.dev):
            rc = self.lib.pvn3d_augment_apply(ptr(rgb), ptr(depth), ptr(labels), ptr(back_rgb), ptr(back_labels), ch,
                                              ptr(back_depth), ptr(params), b, self.h, self.w, DATASETS[self.dataset],
                                              ptr(rgb_out), ptr(depth_out), ptr(stages), ptr(noise), self._ws[1],
                                              self._ws_bytes, self._stream())
        check(rc, "pvn3d_augment_apply")
        return rgb_out, depth_out

    def from_records(self, records: np.ndarray) -> torch.Tensor:
        """explicit records (a numpy structured array of RECORD_DTYPE) -> [B,208] uint8 on the device"""
        if records.dtype != RECORD_DTYPE:
            raise ValueError("FrameAugmenter.from_records: records must be of RECORD_DTYPE")
        raw = np.ascontiguousarray(records).view(np.uint8).reshape(len(records), PARAMS_BYTES)
        return torch.from_numpy(raw.copy()).to(self.dev)


def records(params: torch.Tensor) -> np.ndarray:
    """[B,208] uint8 records -> a numpy structured array of RECORD_DTYPE (host copy; syncs)"""
    raw = params.detach().cpu().numpy()
    return np.ascontiguousarray(raw).view(RECORD_DTYPE).reshape(raw.shape[0])


#: pvn3d_augment_pass_t / pvn3d_augment_params_t (include/pvn3d_b200.h) as numpy dtypes
PASS_DTYPE = np.dtype([("s_factor", "<f8"), ("v_factor", "<f8"), ("sharpen_w", "<f8"), ("sigma", "<f8"),
                       ("sharpen", "<i4"), ("motion", "<i4"), ("angle", "<i4"), ("length", "<i4"),
                       ("gauss", "<i4"), ("ksize", "<i4"), ("noise_sigma", "<i4"), ("extra", "<i4"),
                       ("noise_key", "<u8"), ("extra_key", "<u8")])
RECORD_DTYPE = np.dtype([("kind", "<i4"), ("jitter", "<i4"), ("order", "<i4", (4,)),
                         ("brightness", "<f4"), ("contrast", "<f4"), ("saturation", "<f4"), ("hue", "<f4"),
                         ("n_pass", "<i4"), ("back", "<i4"), ("passes", PASS_DTYPE, (2,))])
assert RECORD_DTYPE.itemsize == PARAMS_BYTES


def probe(op: int, x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """pvn3d_augment_probe: one building block over n inputs (include/pvn3d_b200.h); x and out on one device"""
    n = {0: 3, 1: 3, 2: 3, 3: 3, 4: 3, 5: 2, 6: 2, 7: 3}[op]
    _lib.call("pvn3d_augment_probe", x.device, op, ptr(x), x.numel() // n, ptr(out))
    return out
