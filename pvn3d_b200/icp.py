"""ICP pose refinement -- the reference's `my_icp` (lib/utils/icp/icp.py:141-192), run on the GPU in
float64 by csrc/icp.cu.

    T, distances, i = my_icp(A, B, init_pose, max_iterations=500, tolerance=1e-9)   # drop-in, one object
    ref = IcpRefiner(models, n_cls, batch, n_pts, max_pts=..., min_pts=..., device="cuda")
    poses64, iters, err, refined = ref.refine(pcld, mask, poses, present)          # batched, sync-free

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
    """

    def __init__(self, models, n_cls: int, batch: int, n_pts: int, *, max_pts: int, min_pts: int,
                 max_iter: int = 500, tol: float = 1e-9, device="cuda"):
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
        pts, off = model_table(models, self.n_cls)
        self.lib = _lib.load()
        self.models = IcpModels(pts, off, self.dev)
        self.ws_bytes = int(self.lib.pvn3d_icp_workspace_bytes(self.b, self.n, self.n_cls, self.max_pts))
        if self.ws_bytes == 0:
            raise ValueError("IcpRefiner: problem too large for 32-bit indexing")
        self._ws, self._ws_ptr = _aligned(self.ws_bytes, self.dev)
        shape = (self.b, self.n_cls)
        self.poses = torch.empty(shape + (3, 4), dtype=torch.float64, device=self.dev)
        self.iters = torch.empty(shape, dtype=torch.int32, device=self.dev)
        self.err = torch.empty(shape, dtype=torch.float64, device=self.dev)
        self.refined = torch.empty(shape, dtype=torch.uint8, device=self.dev)

    def pair_tests(self) -> int:
        """diagnostics (synchronises): model points the last refine()'s searches tested"""
        off = self._ws_ptr - self._ws.data_ptr()
        return int(self._ws[off:off + 8].view(torch.int64).item())

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
            rc = self.lib.pvn3d_icp_refine_batch(
                self.models.ptr, ptr(pcld), ptr(mask), b, self.n, self.n_cls, ptr(poses), ptr(present),
                self.max_pts, self.min_pts, self.max_iter, self.tol, ptr(self.poses), ptr(self.iters),
                ptr(self.err), ptr(self.refined), self._ws_ptr, self.ws_bytes,
                cur.cuda_stream)
        check(rc, "pvn3d_icp_refine_batch")
        return self.poses[:b], self.iters[:b], self.err[:b], self.refined[:b]


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
