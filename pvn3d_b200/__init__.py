"""pvn3d_b200 -- H100-native (sm_90a) implementation of PVN3D's per-frame keypoint-voting hot path.

  _ext            drop-in for the reference's `lib.pointnet2_utils._ext` (9 PointNet++ ops)
  pointnet2       host-side mirror of pointnet2_utils / pointnet2_modules / Pointnet2MSG
  meanshift       MeanShiftTorch drop-in (batched Gaussian mean-shift kernels)
  eval_utils      cal_frame_poses / cal_frame_poses_lm / best_fit_transform drop-ins, FramePoseSolver
  pipeline        FramePipeline: both hot paths for a batch of frames, sync-free
  compat          install() the above into an unmodified reference checkout
  dist            frame sharding across GPUs + the single result gather
Everything computes in libpvn3d_b200.so (csrc/*.cu) through the C ABI of include/pvn3d_b200.h.
"""
__version__ = "0.1.0"
