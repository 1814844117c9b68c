"""MeanShiftTorch -- drop-in for the reference class of the same name
(pvn3d/lib/utils/meanshift_pytorch.py:18-51), running the batched sm_90a kernels of
csrc/meanshift.cu through the C ABI.

    ms = MeanShiftTorch(bandwidth=0.08)
    ctr, labels = ms.fit(A)          # A: [n,3] float32 CUDA tensor -> ctr [3] f32, labels [n] bool

Same constructor defaults (bandwidth=0.05, max_iter=300) and return types as the reference; callers
may mutate `labels` and use it as a boolean index (pvn3d_eval_utils.py:86-92).  Beyond the
reference surface, `fit_many` clusters any number of point sets in ONE launch sequence.

No CPU path: a CPU tensor raises (the reference's CPU execution is the *oracle*, see oracle/).
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import torch

from . import _lib
from ._lib import PVN3D_MS_DEBUG_TIMING, check, ms_flags, ptr


class MeanShiftTorch:
    def __init__(self, bandwidth: float = 0.05, max_iter: int = 300, early_exit: bool = False,
                 no_freeze: bool = False, mode: str = None):
        self.bandwidth = bandwidth
        self.stop_thresh = bandwidth * 1e-3  # meanshift_pytorch.py:21 (informational; kernel derives it)
        self.max_iter = max_iter
        #: how the iteration count is decided (include/pvn3d_b200.h, DESIGN.md section 5); every mode returns
        #: the same labels bit for bit and the same centre to well inside the 1e-4 relative parity bar:
        #:   "certified"  (default) only the returned seed + ~60 witness seeds are iterated; a fit whose
        #:                witnesses prove that the reference's stop rule cannot fire before the returned
        #:                seed is within 1e-5*bandwidth of its limit is done, the rest fall back to:
        #:   "early_exit" all seeds, reference stop rule, but a fit also ends once the returned seed is
        #:                stationary (1e-6*bandwidth)
        #:   "strict"     all seeds, reference stop rule: last_iters equals the reference's iteration count
        #:   "no_freeze"  strict + every seed swept at every iteration (the literal reference schedule)
        self.flags = ms_flags(mode, early_exit, no_freeze)
        #: validation: brute-force n^2 density pass instead of the pruned one (PVN3D_MS_BRUTE_DENSITY)
        self.brute_density = False
        self.debug_timing = False
        self.last_iters = None  # iteration count(s) of the last call, device tensor

    # ---- reference surface -------------------------------------------------------------------
    def fit(self, A: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """params: A: [N, 3] -> (C[max_idx] [3], labels [N] bool)"""
        if A.dim() != 2 or A.size(1) != 3:
            raise ValueError("MeanShiftTorch.fit expects an [N, 3] tensor")
        ctrs, labels = self.fit_many([A])
        return ctrs[0], labels[0]

    # ---- batched form ------------------------------------------------------------------------
    def fit_many(self, clouds: Sequence[torch.Tensor]) -> Tuple[torch.Tensor, List[torch.Tensor]]:
        """Cluster every [n_i,3] cloud in one go.  Returns (ctr [F,3], [labels_i bool [n_i]])."""
        if len(clouds) == 0:
            raise ValueError("no clouds")
        dev = clouds[0].device
        if dev.type != "cuda":
            raise RuntimeError("MeanShiftTorch (pvn3d_b200): CUDA tensors only -- no CPU fallback")
        counts = [int(c.size(0)) for c in clouds]
        total = sum(counts)
        nf = len(clouds)
        pts = torch.zeros((max(total, 1), 4), dtype=torch.float32, device=dev)
        if total:
            pts[:total, :3] = torch.cat([c.to(torch.float32) for c in clouds], dim=0)
        starts = [0] * nf
        for i in range(1, nf):
            starts[i] = starts[i - 1] + counts[i - 1]
        fit_start = torch.tensor(starts, dtype=torch.int32, device=dev)
        fit_count = torch.tensor(counts, dtype=torch.int32, device=dev)
        ctr, labels, _, _ = self.fit_segments(pts, fit_start, fit_count, want_labels=True)
        out_labels = [labels[s:s + n].bool() for s, n in zip(starts, counts)]
        return ctr[:, :3], out_labels

    def fit_segments(self, pts4: torch.Tensor, fit_start: torch.Tensor, fit_count: torch.Tensor,
                     want_labels: bool = True):
        """Lowest level: pts4 [cap,4] f32, fit_start/fit_count [F] i32 (all on device).
        Returns (ctr [F,4] (xyz, iterations), labels u8 [cap] or None, max_idx [F], n_in [F])."""
        lib = _lib.load()
        dev = pts4.device
        cap, nf = int(pts4.size(0)), int(fit_start.numel())
        assert pts4.is_contiguous() and pts4.dtype == torch.float32 and pts4.size(1) == 4
        assert fit_start.dtype == torch.int32 and fit_count.dtype == torch.int32
        ctr = torch.empty((nf, 4), dtype=torch.float32, device=dev)
        labels = torch.empty((cap,), dtype=torch.uint8, device=dev) if want_labels else None
        max_idx = torch.empty((nf,), dtype=torch.int32, device=dev)
        n_in = torch.empty((nf,), dtype=torch.int32, device=dev)
        ws_bytes = lib.pvn3d_meanshift_workspace_bytes(cap, nf, int(self.max_iter))
        if ws_bytes == 0:
            raise ValueError("max_iter must be in [0, 4094]")
        ws = torch.empty((ws_bytes + 256,), dtype=torch.uint8, device=dev)
        ws_ptr = (ws.data_ptr() + 255) // 256 * 256
        flags = self.flags | (PVN3D_MS_DEBUG_TIMING if self.debug_timing else 0) | (_lib.PVN3D_MS_BRUTE_DENSITY if self.brute_density else 0)
        self._last_cap_nf = (cap, nf)
        with torch.cuda.device(dev):
            rc = lib.pvn3d_meanshift_fit_batch(
                ptr(pts4), ptr(fit_start), ptr(fit_count), nf, cap, float(self.bandwidth),
                int(self.max_iter), flags, ptr(ctr), ptr(labels), ptr(max_idx), ptr(n_in),
                ws_ptr, ws_bytes, torch.cuda.current_stream(dev).cuda_stream)
        check(rc, "pvn3d_meanshift_fit_batch")
        ws.record_stream(torch.cuda.current_stream(dev))
        self._last_ws = (ws, ws_ptr - ws.data_ptr())   # debug: phase stamps live in the first 1 KB
        self.last_iters = ctr[:, 3]
        return ctr, labels, max_idx, n_in

    def certified_fits(self) -> int:
        """diagnostics (synchronises): fits of the last call closed by the witness kernel"""
        ws, off = self._last_ws
        return int(ws[off:off + 64].view(torch.int32)[_lib.PVN3D_MS_STAT_CERTIFIED].item())

    def last_counts(self) -> torch.Tensor:
        """diagnostics: int32 inlier count of every input point of the last call (indexed like pts4)"""
        ws, off = self._last_ws
        cap, nf = self._last_cap_nf
        o = off + int(_lib.load().pvn3d_meanshift_workspace_counts_offset(cap, nf, int(self.max_iter)))
        return ws[o:o + 4 * cap].view(torch.int32)
