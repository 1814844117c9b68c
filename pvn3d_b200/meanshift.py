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


# --------------------------------------------------------------------------------------------------
# Flat-kernel mean shift (sklearn's MeanShift(bandwidth, bin_seeding=True)), csrc/flat_meanshift.cu
# --------------------------------------------------------------------------------------------------
def flat_mean_shift_batch(X: torch.Tensor, fit_off, bandwidth: float, max_iter: int = 300):
    """Cluster every segment X[fit_off[f]:fit_off[f+1]] in one launch on the current stream.
    X [total,3] float64 contiguous on a CUDA device; fit_off: the F+1 non-decreasing segment offsets on the
    host (a sequence, array or CPU tensor), each segment at most _lib.FLAT_MS_MAX_PTS points -- checked
    here, before anything is launched.  Returns device tensors (labels [total] i32, centres [total,3] f64,
    counts [total] i32, n_clusters [F] i32, n_iter [F] i32): fit f's K = n_clusters[f] centres and their
    member counts are rows fit_off[f] .. fit_off[f]+K-1 (the other rows are unspecified)."""
    import numpy as np

    if not (X.is_cuda and X.dtype == torch.float64 and X.is_contiguous() and X.dim() == 2 and X.size(1) == 3):
        raise ValueError("flat_mean_shift_batch: X must be a contiguous [total,3] float64 CUDA tensor")
    off = fit_off.numpy() if torch.is_tensor(fit_off) else np.asarray(fit_off)
    if off.ndim != 1 or len(off) < 1 or not np.issubdtype(off.dtype, np.integer):
        raise ValueError("flat_mean_shift_batch: fit_off must be F+1 integer offsets")
    sizes = np.diff(off)
    if off[0] < 0 or off[-1] > X.size(0) or (sizes < 0).any():
        raise ValueError(f"flat_mean_shift_batch: fit_off must be non-decreasing within [0, {X.size(0)}]")
    max_fit_pts = int(sizes.max()) if len(sizes) else 0
    if max_fit_pts > _lib.FLAT_MS_MAX_PTS:
        raise ValueError(f"flat_mean_shift_batch: a segment of {max_fit_pts} points, at most "
                         f"{_lib.FLAT_MS_MAX_PTS} per fit")
    if not float(bandwidth) > 0.0:
        raise ValueError(f"bandwidth={bandwidth} must be > 0")
    if int(max_iter) < 0:
        raise ValueError(f"max_iter={max_iter} must be >= 0")
    fit_off = torch.from_numpy(np.ascontiguousarray(off, dtype=np.int32)).to(X.device)
    lib = _lib.load()
    total, n_fits = X.size(0), fit_off.numel() - 1
    labels = torch.empty((total,), dtype=torch.int32, device=X.device)
    centres = torch.empty((total, 3), dtype=torch.float64, device=X.device)
    counts = torch.empty((total,), dtype=torch.int32, device=X.device)
    n_clusters = torch.empty((n_fits,), dtype=torch.int32, device=X.device)
    n_iter = torch.empty((n_fits,), dtype=torch.int32, device=X.device)
    with torch.cuda.device(X.device):
        rc = lib.pvn3d_flat_ms_fit_batch(ptr(X), ptr(fit_off), n_fits, int(max_fit_pts), float(bandwidth),
                                         int(max_iter), ptr(labels), ptr(centres), ptr(counts), ptr(n_clusters),
                                         ptr(n_iter), torch.cuda.current_stream(X.device).cuda_stream)
    check(rc, "pvn3d_flat_ms_fit_batch")
    return labels, centres, counts, n_clusters, n_iter


def flat_mean_shift(X, bandwidth: float, max_iter: int = 300, device="cuda"):
    """sklearn.cluster.mean_shift(X, bandwidth=bandwidth, bin_seeding=True, max_iter=max_iter) on the GPU:
    X [n,3] (array or tensor, used as float64, n <= _lib.FLAT_MS_MAX_PTS) -> (cluster_centers [K,3] f64,
    labels [n] int64, n_iter) as NumPy arrays and an int.  The members of each seed are summed in index
    order, so the result is bit-identical run to run and agrees with sklearn to rounding.  Raises
    ValueError when no point lies within bandwidth of any seed (as sklearn does)."""
    import numpy as np

    a = X.detach().cpu().numpy() if torch.is_tensor(X) else np.asarray(X)
    a = np.ascontiguousarray(a, dtype=np.float64)
    if a.ndim != 2 or a.shape[1] != 3 or len(a) == 0:
        raise ValueError(f"flat_mean_shift: expected non-empty [n,3] points, got shape {a.shape}")
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("flat_mean_shift: CUDA only -- no CPU fallback")
    n = len(a)
    if n > _lib.FLAT_MS_MAX_PTS:
        raise ValueError(f"flat_mean_shift: {n} points, at most {_lib.FLAT_MS_MAX_PTS} per call")
    d_x = torch.from_numpy(a).to(dev)
    labels, centres, _, n_clusters, n_iter = flat_mean_shift_batch(d_x, [0, n], bandwidth, max_iter)
    k = int(n_clusters.cpu()[0])
    if k == 0:
        raise ValueError(f"flat_mean_shift: no point within bandwidth={bandwidth} of any seed")
    return centres[:k].cpu().numpy(), labels.cpu().numpy().astype(np.int64), int(n_iter.cpu()[0])
