"""FramePipeline -- the per-frame keypoint-voting hot path as one device-resident call.

    pipe = FramePipeline("linemod", batch=32)                     # or "ycb", batch=16
    poses, present = pipe.run_host(host_batch)                   # pinned host in, host out (e2e)
    poses, present = pipe.run_device(cld_rgb_nrm, pcld, labels, ctr_of, kp_of)   # resident inputs

One frame = hot path A (Pointnet2MSG.forward on [N,9]) + hot path B (cal_frame_poses* on that
frame's votes), the unit BASELINE.json's frames/sec counts (SURVEY section 8d).  Both run on the
current CUDA stream with no host synchronisation; the only copies are the ones run_host() makes.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch

from . import fixtures
from .eval_utils import FramePoseSolver
from .mlp import FusedPointnet2MSG
from .testing import seeded_pointnet2msg


class FramePipeline:
    def __init__(self, shape: str, batch: int, n_points: int = fixtures.N_SAMPLE_POINTS, device="cuda",
                 lm_obj_id: int = 1, early_exit: bool = False, model: Optional[torch.nn.Module] = None,
                 allow_tf32: bool = True, engine: str = "fused", ms_mode: Optional[str] = None,
                 overlap: bool = True, bandwidth: float = 0.08, fps_chunk: int = 0, pose_stream: bool = True,
                 reserve_levels: Optional[int] = None):
        self.dev = torch.device(device)
        self.shape, self.b, self.n, self.k = shape, int(batch), int(n_points), fixtures.N_KEYPOINTS
        self.model = (model if model is not None else seeded_pointnet2msg(0, 1)).to(self.dev).eval()
        #: "fused"  = hot path A entirely on libpvn3d_b200 (wgmma shared MLPs, grouping/interpolation fused
        #:            into the operand producers -- pvn3d_b200.mlp.FusedPointnet2MSG)
        #: "modules" = the Pointnet2MSG module graph on the library's `_ext` ops with cuDNN/cuBLAS MLPs
        self.engine = engine
        self.fused = FusedPointnet2MSG(self.model, self.dev) if engine == "fused" else None
        if shape == "linemod":
            self.n_cls = 2
            mesh = fixtures.mesh_kps_table_lm(lm_obj_id)
            self.solver = FramePoseSolver(self.b, self.n, self.k, 2, mesh, None, False, device=self.dev,
                                          early_exit=early_exit, mode=ms_mode, bandwidth=bandwidth)
        elif shape == "ycb":
            self.n_cls = fixtures.YCB_N_CLASSES
            self.solver = FramePoseSolver(self.b, self.n, self.k, self.n_cls, fixtures.mesh_kps_table_ycb(),
                                          fixtures.radius_thresholds_ycb(), True, device=self.dev,
                                          early_exit=early_exit, mode=ms_mode, bandwidth=bandwidth)
        else:
            raise ValueError(shape)
        self.allow_tf32 = allow_tf32
        # device staging buffers for run_host(): two sets, so that the H2D copies of call i (on their own
        # stream) run under the kernels of call i-1
        f32 = dict(dtype=torch.float32, device=self.dev)
        self._sets = [dict(cld_rgb_nrm=torch.empty((self.b, self.n, 9), **f32),
                           pcld=torch.empty((self.b, self.n, 3), **f32),
                           labels=torch.empty((self.b, self.n), dtype=torch.int32, device=self.dev),
                           ctr_of=torch.empty((self.b, self.n, 3), **f32),
                           kp_of=torch.empty((self.b, self.k, self.n, 3), **f32)) for _ in range(2)]
        self._set_free = [None, None]     # event: the kernels that last read the set are done
        self._turn = 0
        self._copy_stream = torch.cuda.Stream(self.dev)
        #: hot path B (votes -> poses) does not read hot path A's features (the votes come from the network
        #: heads, synthetic here): it runs on its own stream, so its many small kernels fill the SMs that the
        #: latency-bound furthest-point sampling of path A (one CTA per frame) leaves idle
        self.overlap = bool(overlap)
        self._pose_stream = torch.cuda.Stream(self.dev) if (self.overlap and pose_stream) else None
        #: look-ahead: when the caller names the NEXT batch (run_device(..., next_cloud=) / run_host(hb, next_hb)),
        #: its coordinate-only half of hot path A (furthest-point sampling: 3708 dependent iterations on one CTA
        #: per frame, plus ball queries and 3-NN) runs on a third stream UNDER the shared MLPs of the current
        #: batch.  The sampling kernels are launched `fps_chunk` frames at a time (0: the whole batch) and the
        #: persistent MLP kernels of the first `reserve_levels` SA levels leave that many SMs free
        #: (PVN3D_MLP_RESERVE_SMS), so neither side waits for an SM; the sampling (2 ms for 32 frames side by side) is
        #: over by then and the later, larger half of the MLPs takes the whole machine.  (Round 2 first used 16-frame
        #: chunks under all layers: 2 x 2 ms of sampling -- hidden while the MLPs took 3.4 ms, the critical path once
        #: they took 2.8.)
        # 32 x 12288: the MLPs (2.7 ms) outlast the sampling (2.1 ms) -> reserve under SA1-2 only (3.93 vs 4.38 ms per step
        # with all levels reserving).  Smaller batches / larger clouds: the sampling is the critical path and a sampling
        # kernel that finds every SM taken by a full-width layer waits for it -> reserve under every layer
        if reserve_levels is None:
            reserve_levels = 2 if (self.b >= 24 and self.n <= 16384) else 5
        self.reserve_levels = int(reserve_levels)
        self.fps_chunk = max(1, min(fps_chunk if fps_chunk > 0 else self.b, self.b))
        # high priority: a sampling CTA needs a whole SM (512 threads, ~56 K registers, 147 KB shared memory); when
        # an SM drains, it must win it before the thousands of small CTAs of hot path B refill it
        self._geo_stream = torch.cuda.Stream(self.dev, priority=-1) if self.overlap else None
        self._plan = None
        self._plan_host = None            # id of the pinned host batch the look-ahead plan was computed for
        self._staged = [None, None]       # (id of the pinned host batch uploaded into the set, upload event)
        self.d_cloud, self.d_pcld, self.d_labels, self.d_ctr_of, self.d_kp_of = (
            self._sets[0][k] for k in ("cld_rgb_nrm", "pcld", "labels", "ctr_of", "kp_of"))
        # pinned result buffers, one pair per staging set: call i+1 must not overwrite what call i returned
        # before the caller has synchronised and read it
        self._h_out = [(torch.empty((self.b, self.n_cls, 3, 4), dtype=torch.float32).pin_memory(),
                        torch.empty((self.b, self.n_cls), dtype=torch.uint8).pin_memory()) for _ in range(2)]
        self.h_poses, self.h_present = self._h_out[0]
        self.features = None

    def h2d_bytes(self) -> int:
        return sum(t.numel() * t.element_size() for t in
                   (self.d_cloud, self.d_pcld, self.d_labels, self.d_ctr_of, self.d_kp_of))

    def d2h_bytes(self) -> int:
        return self.h_poses.numel() * 4 + self.h_present.numel()

    @staticmethod
    def pin_batch(batch: Dict[str, np.ndarray]) -> Dict[str, torch.Tensor]:
        return {k: torch.from_numpy(np.ascontiguousarray(v)).pin_memory() for k, v in batch.items()}

    @torch.no_grad()
    def run_device(self, cld_rgb_nrm, pcld, labels, ctr_of, kp_of, next_cloud=None):
        """inputs resident in HBM; returns device views (poses [B,n_cls,3,4], present [B,n_cls]).
        next_cloud: the cld_rgb_nrm tensor of the batch the NEXT call will process (or (tensor, event that
        signals its upload)): its geometry plan is computed on a side stream during this call."""
        cur = torch.cuda.current_stream(self.dev)
        ready = torch.cuda.Event()
        ready.record(cur)
        if self._pose_stream is not None:
            self._pose_stream.wait_event(ready)          # inputs (and the previous reader of the outputs) are done
            with torch.cuda.stream(self._pose_stream):
                poses, present, _, _ = self.solver.solve(pcld, labels, ctr_of, kp_of)   # hot path B
                solved = torch.cuda.Event()
                solved.record(self._pose_stream)
        if self.fused is not None:
            plan, self._plan = self._plan, None
            if plan is not None and plan.key != (cld_rgb_nrm.data_ptr(), tuple(cld_rgb_nrm.shape)):
                plan = None                                               # the look-ahead was for another batch
            if plan is None:
                plan = self.fused.geometry(cld_rgb_nrm)                   # no look-ahead: geometry first, whole GPU
            else:
                # The plan's tensors were allocated on the sampling stream and are read here on `cur`.  No
                # record_stream() is needed (and its deferred frees made the caching allocator call cudaMalloc
                # every few steps): the plan is dropped when this call returns, its blocks go back to the
                # sampling stream's pool, and the next allocation from that pool is the sampling of call i+1,
                # which waits for `ready` of call i+1 -- recorded on `cur` after everything enqueued here.
                cur.wait_event(plan.done)
            reserve = 0
            if next_cloud is not None and self.overlap:
                nc, uploaded = next_cloud if isinstance(next_cloud, tuple) else (next_cloud, None)
                g = self._geo_stream
                g.wait_event(ready)
                if uploaded is not None:
                    g.wait_event(uploaded)
                with torch.cuda.stream(g):
                    nplan = self.fused.sampling(nc, fps_chunk=self.fps_chunk)
                    nplan.done = torch.cuda.Event()
                    nplan.done.record(g)
                self._plan = nplan
                reserve = min(self.fps_chunk, nc.size(0))
            self.features = self.fused.features(cld_rgb_nrm, plan, reserve_sms=reserve,
                                                reserve_levels=self.reserve_levels)        # hot path A: [B,128,N]
        else:
            prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
            torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = self.allow_tf32
            try:
                self.features = self.model(cld_rgb_nrm)
            finally:
                torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
        if self._pose_stream is not None:
            cur.wait_event(solved)
        else:
            poses, present, _, _ = self.solver.solve(pcld, labels, ctr_of, kp_of)   # hot path B
        return poses, present

    def _upload(self, hb: Dict[str, torch.Tensor], turn: int):
        st = self._sets[turn]
        b = hb["pcld"].shape[0]
        with torch.cuda.stream(self._copy_stream):
            if self._set_free[turn] is not None:
                self._copy_stream.wait_event(self._set_free[turn])
            # the cloud goes first and gets its own event: the look-ahead sampling (4 ms on the critical path of the NEXT
            # step) needs nothing else, and must not wait for the 45 MB of votes behind it
            st["cld_rgb_nrm"][:b].copy_(hb["cld_rgb_nrm"], non_blocking=True)
            cloud_up = torch.cuda.Event()
            cloud_up.record(self._copy_stream)
            for key in ("pcld", "labels", "ctr_of", "kp_of"):
                st[key][:b].copy_(hb[key], non_blocking=True)
            uploaded = torch.cuda.Event()
            uploaded.record(self._copy_stream)
        self._staged[turn] = (id(hb), uploaded)
        self._cloud_up = cloud_up
        return uploaded

    @torch.no_grad()
    def run_host(self, hb: Dict[str, torch.Tensor], next_hb: Optional[Dict[str, torch.Tensor]] = None):
        """hb: pinned host tensors (pin_batch).  H2D copies, both hot paths, D2H of the poses; the
        caller synchronises the stream before reading the returned pinned host tensors.  The copies
        go through a second stream into one of two staging sets: back-to-back calls overlap the
        upload of call i with the kernels of call i-1.  The returned pinned buffers alternate too: the
        result of call i stays valid until call i+2.
        next_hb: the batch the NEXT call will process: it is uploaded now (into the other staging set) and its
        geometry plan is computed under this call's shared MLPs (see run_device)."""
        b = hb["pcld"].shape[0]
        turn = self._turn
        self._turn ^= 1
        st = self._sets[turn]
        cur = torch.cuda.current_stream(self.dev)
        tag = self._staged[turn]
        if self._plan is not None and self._plan_host != id(hb):
            # the look-ahead named another batch: drop its plan (the staging buffer it was computed from has this
            # call's address) and let the sampler finish reading that buffer before it is overwritten
            self._copy_stream.wait_event(self._plan.done)
            self._plan = None
        self._plan_host = None
        uploaded = tag[1] if (tag is not None and tag[0] == id(hb)) else self._upload(hb, turn)
        self._staged[turn] = None
        cur.wait_event(uploaded)
        next_cloud = None
        if next_hb is not None and self.overlap and self.fused is not None:
            self._upload(next_hb, turn ^ 1)
            next_cloud = (self._sets[turn ^ 1]["cld_rgb_nrm"][:next_hb["pcld"].shape[0]], self._cloud_up)
            self._plan_host = id(next_hb)
        poses, present = self.run_device(st["cld_rgb_nrm"][:b], st["pcld"][:b], st["labels"][:b],
                                         st["ctr_of"][:b], st["kp_of"][:b], next_cloud=next_cloud)
        done = torch.cuda.Event()
        done.record(cur)
        self._set_free[turn] = done
        h_poses, h_present = self._h_out[turn]
        h_poses[:b].copy_(poses, non_blocking=True)
        h_present[:b].copy_(present, non_blocking=True)
        return h_poses[:b], h_present[:b]
