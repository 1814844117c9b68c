"""ctypes binding of libpvn3d_b200.so -- the only way Python reaches the kernels.

The library is the product: if it is missing or cannot be loaded this module raises, and every
op built on it raises with it.  There is no PyTorch / CPU fallback anywhere in this package.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_size_t, c_uint, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpvn3d_b200.so")

PVN3D_MS_STRICT = 0
PVN3D_MS_EARLY_EXIT = 1
PVN3D_MS_NO_FREEZE = 2
PVN3D_MS_DEBUG_TIMING = 4
PVN3D_MS_CERTIFIED = 8
PVN3D_MS_BRUTE_DENSITY = 16
PVN3D_MS_STAT_CERTIFIED = 8   # int32 word of the mean-shift workspace: fits closed by the witness kernel

#: mode name -> flags of the mean-shift iteration (include/pvn3d_b200.h)
MS_MODES = {"certified": PVN3D_MS_CERTIFIED | PVN3D_MS_EARLY_EXIT, "early_exit": PVN3D_MS_EARLY_EXIT,
            "strict": PVN3D_MS_STRICT, "no_freeze": PVN3D_MS_NO_FREEZE}
MS_DEFAULT_MODE = "certified"


def ms_flags(mode=None, early_exit=False, no_freeze=False) -> int:
    """flags from a mode name; the round-1 keyword switches (early_exit / no_freeze) still select their modes"""
    if mode is None:
        mode = "no_freeze" if no_freeze else ("early_exit" if early_exit else MS_DEFAULT_MODE)
    if mode not in MS_MODES:
        raise ValueError(f"unknown mean-shift mode {mode!r}: one of {sorted(MS_MODES)}")
    return MS_MODES[mode]

_ERR_NAMES = {-1: "invalid argument", -2: "unsupported size", -3: "CUDA error", -4: "workspace too small"}

class MlpLayer(ctypes.Structure):
    """pvn3d_mlp_layer_t (include/pvn3d_b200.h)"""
    _fields_ = [("w", c_void_p), ("bias", c_void_p), ("k_pad", c_int), ("n_pad", c_int)]


class LossArgs(ctypes.Structure):
    """pvn3d_loss_args_t (include/pvn3d_b200.h)"""
    _fields_ = [("seg", c_void_p), ("seg_target", c_void_p), ("seg_rows", ctypes.c_longlong), ("n_cls", c_int),
                ("seg_inner", c_int), ("gamma", c_float), ("seg_mean", c_int), ("kp_pred", c_void_p),
                ("kp_targ", c_void_p), ("n_kp", c_int), ("ctr_pred", c_void_p), ("ctr_targ", c_void_p),
                ("n_ctr", c_int), ("labels", c_void_p), ("b", c_int), ("n", c_int), ("ok", c_void_p),
                ("w_seg", c_float), ("w_kp", c_float), ("w_ctr", c_float)]


# name -> (restype, argtypes); mirrors include/pvn3d_b200.h one to one
_P = c_void_p
_SIGNATURES = {
    "pvn3d_version": (c_int, []),
    "pvn3d_strerror": (c_char_p, [c_int]),
    "pvn3d_last_cuda_error": (c_char_p, []),
    "pvn3d_device_sm_count": (c_int, [_P, _P, _P]),
    "pvn3d_launch_count": (ctypes.c_ulonglong, []),
    "pvn3d_furthest_point_sampling": (c_int, [_P, c_int, c_int, c_int, _P, _P]),
    "pvn3d_gather_points": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P, _P]),
    "pvn3d_gather_xyz": (c_int, [_P, _P, c_int, c_int, c_int, _P, _P]),
    "pvn3d_gather_points_grad": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P, _P]),
    "pvn3d_ball_query": (c_int, [_P, _P, c_int, c_int, c_int, c_float, c_int, _P, _P]),
    "pvn3d_group_points": (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, _P, _P]),
    "pvn3d_group_points_grad": (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, _P, _P]),
    "pvn3d_three_nn": (c_int, [_P, _P, c_int, c_int, c_int, _P, _P, _P]),
    "pvn3d_three_nn_grid_supported": (c_int, [c_int, c_int]),
    "pvn3d_three_nn_weights_levels": (c_int, [c_int, _P, _P, _P, _P, c_int, _P, _P, _P, _P]),
    "pvn3d_ball_grid_supported": (c_int, [c_int, c_int, c_int, c_int]),
    "pvn3d_ball_query2_levels": (c_int, [c_int, _P, _P, _P, _P, c_int, _P, _P, _P, _P, _P, _P, _P]),
    "pvn3d_three_interpolate": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, _P, _P]),
    "pvn3d_three_interpolate_grad": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, _P, _P]),
    "pvn3d_transpose_cn_to_nc": (c_int, [_P, c_int, c_int, c_int, _P, _P]),
    "pvn3d_transpose_nc_to_cn": (c_int, [_P, c_int, c_int, c_int, _P, _P]),
    "pvn3d_query_and_group": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_float, c_int, _P, _P, _P]),
    "pvn3d_query_and_group2": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_float, c_int, _P, _P, c_float, c_int, _P, _P, _P]),
    "pvn3d_three_nn_interpolate": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, _P, c_int, c_int, _P, _P, _P]),
    "pvn3d_mlp_dense": (c_int, [_P, c_int, c_int, ctypes.c_longlong, _P, _P, c_int, c_int, c_int, _P, c_int, c_int, _P]),
    "pvn3d_mlp_dense_frame_bias": (c_int, [_P, c_int, c_int, ctypes.c_longlong, c_int, _P, _P, c_int, c_int, c_int, _P, c_int, c_int, _P]),
    "pvn3d_mlp_dense_sum32": (c_int, [_P, c_int, c_int, ctypes.c_longlong, _P, _P, c_int, c_int, c_int, _P, c_int, c_int, _P]),
    "pvn3d_sa_factor_table": (c_int, [_P, _P, c_int, c_int, ctypes.c_longlong, c_int, _P, _P]),
    "pvn3d_sa_centre_term": (c_int, [_P, _P, _P, ctypes.c_longlong, c_int, _P, _P]),
    "pvn3d_mlp_sa_fact2": (c_int, [_P, _P, c_int, c_int, _P, c_int, c_int, c_int, c_int, _P, _P, c_int, c_int, _P, c_int,
                                   c_int, _P]),
    "pvn3d_mlp_sa_fact2_supported": (c_int, [_P, _P, c_int]),
    "pvn3d_mlp_sa_fact2w": (c_int, [_P, _P, c_int, c_int, _P, c_int, c_int, c_int, c_int, _P, _P, c_int, c_int, _P, c_int,
                                    c_int, _P]),
    "pvn3d_mlp_sa_fact2w_supported": (c_int, [_P, _P, c_int]),
    "pvn3d_mlp_fp2": (c_int, [_P, c_int, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P, _P, c_int, _P, c_int, c_int, _P]),
    "pvn3d_mlp_fp2_supported": (c_int, [_P, _P]),
    "pvn3d_mlp_fp_fact2": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, _P, _P, c_int, _P, _P]),
    "pvn3d_mlp_fp_fact2_supported": (c_int, [_P, _P]),
    "pvn3d_mlp_fp_fact2_rows": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, _P, _P, c_int, _P, c_int, c_int, _P]),
    "pvn3d_gather_pixel_rows": (c_int, [_P, c_int, c_int, ctypes.c_longlong, _P, c_int, _P, c_int, c_int, _P]),
    "pvn3d_mlp_dense_bf16": (c_int, [_P, c_int, c_int, ctypes.c_longlong, _P, _P, c_int, c_int, c_int, _P, c_int, c_int, _P]),
    "pvn3d_mlp_dense_frame_bias_bf16": (c_int, [_P, c_int, c_int, ctypes.c_longlong, c_int, _P, _P, c_int, c_int, c_int, _P,
                                                c_int, c_int, _P]),
    "pvn3d_mlp_dense_sum32_bf16": (c_int, [_P, c_int, c_int, ctypes.c_longlong, _P, _P, c_int, c_int, c_int, _P, c_int, c_int,
                                           _P]),
    "pvn3d_mlp_fp_fact2_rows_bf16": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, _P, _P, c_int, _P, c_int, c_int, _P]),
    "pvn3d_gather_pixel_rows_bf16": (c_int, [_P, c_int, c_int, c_int, ctypes.c_longlong, _P, c_int, _P, c_int, c_int, _P]),
    "pvn3d_psp_tail_rows": (c_int, [_P, c_int, c_int, c_int, _P, c_int, _P, _P, _P, c_int, _P, c_int, c_int, _P]),
    "pvn3d_psp_tail_rows_bf16": (c_int, [_P, c_int, c_int, c_int, _P, c_int, _P, _P, _P, c_int, _P, c_int, c_int, _P]),
    "pvn3d_psp_tail_supported": (c_int, [_P, _P]),
    "pvn3d_three_nn_weights": (c_int, [_P, ctypes.c_longlong, _P, _P]),
    "pvn3d_seg_argmax": (c_int, [_P, ctypes.c_longlong, c_int, _P, _P]),
    "pvn3d_pose_add_adds_workspace_bytes": (c_size_t, [c_int, c_int]),
    "pvn3d_pose_add_adds": (c_int, [_P, _P, c_int, _P, c_int, _P, _P, _P, c_size_t, _P]),
    "pvn3d_frame_add_adds_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "pvn3d_frame_add_adds": (c_int, [_P, _P, c_int, _P, _P, c_int, c_int, _P, _P, c_int, _P, _P, _P, c_size_t, _P]),
    "pvn3d_meanshift_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "pvn3d_meanshift_workspace_counts_offset": (c_size_t, [c_int, c_int, c_int]),
    "pvn3d_meanshift_fit_batch": (c_int, [_P, _P, _P, c_int, c_int, c_double, c_int, c_uint, _P, _P, _P, _P, _P, c_size_t, _P]),
    "pvn3d_best_fit_transform_batch": (c_int, [_P, _P, _P, c_int, c_int, _P, _P]),
    "pvn3d_frame_poses_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "pvn3d_frame_poses_ms_workspace_offset": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "pvn3d_frame_poses_batch": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_int, _P, _P, c_int, c_double, c_int, c_uint, _P, _P, _P, _P, _P, c_size_t, _P]),
    "pvn3d_icp_models_bytes": (c_size_t, [c_int, c_int]),
    "pvn3d_icp_build_models": (c_int, [_P, _P, c_int, c_int, _P, c_size_t, _P]),
    "pvn3d_icp_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "pvn3d_icp_refine_batch": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P, _P, c_int, c_int, c_int, c_double, _P, _P, _P, _P,
                                       _P, c_size_t, _P]),
    "pvn3d_icp_fit": (c_int, [_P, c_int, _P, c_int, _P, c_int, c_double, _P, _P, _P, _P, _P, c_size_t, _P]),
    "pvn3d_flat_ms_fit_batch": (c_int, [_P, _P, c_int, c_int, c_double, c_int, _P, _P, _P, _P, _P, _P]),
    "pvn3d_icp_clustered_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "pvn3d_icp_refine_batch_clustered": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P, _P, c_int, c_int, c_int, c_double,
                                                 c_double, c_int, _P, _P, _P, _P, _P, _P, c_size_t, _P]),
    "pvn3d_depth_to_cloud": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P, _P, _P]),
    "pvn3d_label_fill_workspace_bytes": (c_size_t, [c_int, c_int]),
    "pvn3d_label_fill": (c_int, [_P, _P, c_int, _P, _P, c_int, c_int, _P, _P, _P, c_size_t, _P]),
    "pvn3d_frame_sample_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "pvn3d_frame_sample": (c_int, [_P, _P, _P, c_int, _P, c_int, c_int, c_int, ctypes.c_ulonglong, _P, ctypes.c_longlong,
                                   _P, _P, _P, _P, _P, c_size_t, _P]),
    "pvn3d_knn_normals_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "pvn3d_knn_normals": (c_int, [_P, _P, c_int, _P, c_int, c_int, _P, _P, ctypes.c_longlong, _P, _P, _P, _P, c_size_t,
                                  _P]),
    "pvn3d_depth_fill_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "pvn3d_depth_fill": (c_int, [_P, _P, c_float, c_int, c_int, c_int, _P, _P, _P, _P, c_size_t, _P]),
    "pvn3d_augment_draw": (c_int, [ctypes.c_ulonglong, _P, c_int, c_int, _P, _P]),
    "pvn3d_augment_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "pvn3d_augment_apply": (c_int, [_P, _P, _P, _P, _P, c_int, _P, _P, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P,
                                    c_size_t, _P]),
    "pvn3d_augment_probe": (c_int, [c_int, _P, ctypes.c_longlong, _P, _P]),
    "pvn3d_train_targets":(c_int, [_P, _P, _P, _P, c_int, c_int, c_int, _P, _P, c_int, c_int, _P, _P, _P, _P, _P]),
    "pvn3d_train_loss_workspace_bytes": (c_size_t, [ctypes.POINTER(LossArgs)]),
    "pvn3d_train_loss_forward": (c_int, [ctypes.POINTER(LossArgs), _P, _P, _P, _P, _P, _P, c_size_t, _P]),
    "pvn3d_train_loss_backward": (c_int, [ctypes.POINTER(LossArgs), _P, _P, _P, _P, _P, _P, _P, c_size_t, _P]),
    "pvn3d_vis_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "pvn3d_vis_draw_poses": (c_int, [_P, c_int, c_int, c_int, _P, _P, c_int, c_int, _P, c_int, _P, _P, c_int, _P,
                                     c_double, _P, c_int, _P, c_size_t, _P]),
    "pvn3d_vis_draw_p2ds": (c_int, [_P, c_int, c_int, _P, c_int, c_int, c_uint, _P, c_size_t, _P]),
    "pvn3d_render_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "pvn3d_render_meshes": (c_int, [_P, _P, _P, _P, _P, c_int, c_int, c_int, _P, c_int, _P, _P, c_int, c_int, c_int,
                                    c_double, _P, _P, _P, _P, _P, _P, c_size_t, _P]),
    "pvn3d_ordered_grad_workspace_bytes":(c_size_t, [c_int, c_int, ctypes.c_longlong]),
    "pvn3d_gather_points_grad_ordered": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P, _P, c_size_t, _P]),
    "pvn3d_group_points_grad_ordered": (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, _P, _P, c_size_t, _P]),
    "pvn3d_three_interpolate_grad_ordered": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, _P, _P, c_size_t, _P]),
    "pvn3d_adaptive_avg_pool2d_backward": (c_int, [_P, ctypes.c_longlong, c_int, c_int, c_int, c_int, _P, _P]),
    "pvn3d_upsample_bilinear2d_backward": (c_int, [_P, ctypes.c_longlong, c_int, c_int, c_int, c_int, c_int, c_double,
                                                   c_double, _P, _P]),
    "pvn3d_group_points_16": (c_int, [c_int, _P, _P, c_int, c_int, c_int, c_int, c_int, _P, _P]),
    "pvn3d_group_points_grad_16": (c_int, [c_int, _P, _P, c_int, c_int, c_int, c_int, c_int, _P, _P, _P]),
    "pvn3d_three_interpolate_16": (c_int, [c_int, _P, _P, _P, c_int, c_int, c_int, c_int, _P, _P]),
    "pvn3d_three_interpolate_grad_16": (c_int, [c_int, _P, _P, _P, c_int, c_int, c_int, c_int, _P, _P, _P]),
    "pvn3d_group_points_grad_ordered_16": (c_int, [c_int, _P, _P, c_int, c_int, c_int, c_int, c_int, _P, _P, c_size_t,
                                                   _P]),
    "pvn3d_three_interpolate_grad_ordered_16": (c_int, [c_int, _P, _P, _P, c_int, c_int, c_int, c_int, _P, _P, c_size_t,
                                                        _P]),
    "pvn3d_adaptive_avg_pool2d_backward_16": (c_int, [c_int, _P, ctypes.c_longlong, c_int, c_int, c_int, c_int, _P, _P]),
    "pvn3d_upsample_bilinear2d_backward_16": (c_int, [c_int, _P, ctypes.c_longlong, c_int, c_int, c_int, c_int, c_int,
                                                      c_double, c_double, _P, _P]),
}
FLAT_MS_MAX_PTS = 4096   # PVN3D_FLAT_MS_MAX_PTS
EXPORTED_SYMBOLS = tuple(_SIGNATURES)
PVN3D_F16, PVN3D_BF16 = 1, 2   # dtype codes of the *_16 entry points

_lib = None


class Pvn3dError(RuntimeError):
    pass


def load() -> ctypes.CDLL:
    """dlopen the kernel library (once).  Raises Pvn3dError when it is absent: build it with
    `python -m pvn3d_b200.build` (or __graft_entry__.build())."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise Pvn3dError(
            f"{LIB_PATH} not found: the sm_90a kernel library is not built "
            "(run `python -m pvn3d_b200.build`); pvn3d_b200 has no CPU / PyTorch fallback")
    try:
        lib = ctypes.CDLL(LIB_PATH)
    except OSError as e:  # pragma: no cover
        raise Pvn3dError(f"cannot load {LIB_PATH}: {e}") from e
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the header and the library disagree
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc == 0:
        return
    lib = load()
    msg = _ERR_NAMES.get(rc, f"error {rc}")
    if rc == -3:
        detail = lib.pvn3d_last_cuda_error()
        msg += f": {detail.decode() if detail else '?'}"
    raise Pvn3dError(f"{what}: {msg}")


def call(fn_name: str, dev, *args) -> None:
    """fn_name(*args, stream) with `dev` the current device and stream its current stream; raises Pvn3dError on a
    non-zero return code"""
    import torch

    lib = load()
    with torch.cuda.device(dev):
        rc = getattr(lib, fn_name)(*args, torch.cuda.current_stream(dev).cuda_stream)
    check(rc, fn_name)


def ptr(t) -> int:
    """device/host address of a torch tensor (0 for None)"""
    return 0 if t is None else t.data_ptr()


def stream_ptr(device=None) -> int:
    import torch

    return torch.cuda.current_stream(device).cuda_stream
