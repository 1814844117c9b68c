"""Drop-in for the reference's pybind11 module `lib.pointnet2_utils._ext`.

Same nine functions, argument order, dtypes, output allocation and error text as
pvn3d/_ext-src/src/bindings.cpp:6-19 and the host wrappers in pvn3d/_ext-src/src/*.cpp, but every
call lands in a hand-written sm_90a kernel of libpvn3d_b200.so through the C ABI
(include/pvn3d_b200.h).  Install it with `pvn3d_b200.compat.install()` and the reference's
`pointnet2_utils.py` / `pointnet2_modules.py` / `demo.py` / `train_*.py` run on it unchanged.

Contract kept from the reference (SURVEY section 8b):
  * inputs must be contiguous float32 / int32 tensors (RuntimeError "<name> must be a contiguous
    tensor" etc., utils.h:5-25); CPU tensors raise "CPU not supported" (e.g. ball_query.cpp:28);
  * the callee allocates and returns new tensors, inputs are never written;
  * launches go to the caller's current stream, asynchronously, no syncs; the input's device is
    made current for the call (the reference has no device guard -- added here).
Divergence, on purpose: three_interpolate_grad computes the correct gradient (the reference host
wrapper launches the forward kernel, interpolate.cpp:89-93 -- a training-only bug).
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import check, ptr


def _chk_contig(x, name):
    if not x.is_contiguous():
        raise RuntimeError(f"{name} must be a contiguous tensor")


def _chk_float(x, name):
    if x.dtype != torch.float32:
        raise RuntimeError(f"{name} must be a float tensor")


def _chk_int(x, name):
    if x.dtype != torch.int32:
        raise RuntimeError(f"{name} must be an int tensor")


def _chk_cuda(x, name):
    if not x.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor")


def _need_cuda(x):
    if not x.is_cuda:
        raise RuntimeError("CPU not supported")


def _call(fn_name, dev, *args):
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = getattr(lib, fn_name)(*args, torch.cuda.current_stream(dev).cuda_stream)
    check(rc, fn_name)


def furthest_point_sampling(points: torch.Tensor, nsamples: int) -> torch.Tensor:
    """sampling.cpp:65-86 -- points [B,N,3] f32 -> idx [B,nsamples] i32"""
    _chk_contig(points, "points")
    _chk_float(points, "points")
    _need_cuda(points)
    b, n = points.size(0), points.size(1)
    out = torch.empty((b, nsamples), dtype=torch.int32, device=points.device)
    _call("pvn3d_furthest_point_sampling", points.device, ptr(points), b, n, int(nsamples), ptr(out))
    return out


def gather_points(points: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """sampling.cpp:15-38 -- points [B,C,N], idx [B,M] -> [B,C,M]"""
    _chk_contig(points, "points")
    _chk_contig(idx, "idx")
    _chk_float(points, "points")
    _chk_int(idx, "idx")
    if points.is_cuda:
        _chk_cuda(idx, "idx")
    _need_cuda(points)
    b, c, n = points.shape
    m = idx.size(1)
    out = torch.empty((b, c, m), dtype=torch.float32, device=points.device)
    _call("pvn3d_gather_points", points.device, ptr(points), ptr(idx), b, c, n, m, ptr(out))
    return out


def gather_xyz(xyz: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """xyz [B,N,3] f32, idx [B,M] i32 -> new_xyz [B,M,3] (point-major gather_operation, pointnet2_modules.py:47-53)"""
    _chk_contig(xyz, "xyz"); _chk_contig(idx, "idx")
    _chk_float(xyz, "xyz"); _chk_int(idx, "idx")
    _need_cuda(xyz)
    b, n, _ = xyz.shape
    m = idx.size(1)
    out = torch.empty((b, m, 3), dtype=torch.float32, device=xyz.device)
    _call("pvn3d_gather_xyz", xyz.device, ptr(xyz), ptr(idx), b, n, m, ptr(out))
    return out


def gather_points_grad(grad_out: torch.Tensor, idx: torch.Tensor, n: int) -> torch.Tensor:
    """sampling.cpp:40-63"""
    _chk_contig(grad_out, "grad_out")
    _chk_contig(idx, "idx")
    _chk_float(grad_out, "grad_out")
    _chk_int(idx, "idx")
    if grad_out.is_cuda:
        _chk_cuda(idx, "idx")
    _need_cuda(grad_out)
    b, c, m = grad_out.shape
    out = torch.empty((b, c, int(n)), dtype=torch.float32, device=grad_out.device)
    _call("pvn3d_gather_points_grad", grad_out.device, ptr(grad_out), ptr(idx), b, c, int(n), m, ptr(out))
    return out


def ball_query(new_xyz: torch.Tensor, xyz: torch.Tensor, radius: float, nsample: int) -> torch.Tensor:
    """ball_query.cpp:8-32 -- NOTE the argument order: centres first."""
    _chk_contig(new_xyz, "new_xyz")
    _chk_contig(xyz, "xyz")
    _chk_float(new_xyz, "new_xyz")
    _chk_float(xyz, "xyz")
    if new_xyz.is_cuda:
        _chk_cuda(xyz, "xyz")
    _need_cuda(new_xyz)
    b, n = xyz.size(0), xyz.size(1)
    m = new_xyz.size(1)
    idx = torch.empty((new_xyz.size(0), m, int(nsample)), dtype=torch.int32, device=new_xyz.device)
    _call("pvn3d_ball_query", new_xyz.device, ptr(new_xyz), ptr(xyz), b, n, m, float(radius), int(nsample), ptr(idx))
    return idx


def group_points(points: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """group_points.cpp:12-35 -- points [B,C,N], idx [B,M,S] -> [B,C,M,S]"""
    _chk_contig(points, "points")
    _chk_contig(idx, "idx")
    _chk_float(points, "points")
    _chk_int(idx, "idx")
    if points.is_cuda:
        _chk_cuda(idx, "idx")
    _need_cuda(points)
    b, c, n = points.shape
    m, s = idx.size(1), idx.size(2)
    out = torch.empty((b, c, m, s), dtype=torch.float32, device=points.device)
    _call("pvn3d_group_points", points.device, ptr(points), ptr(idx), b, c, n, m, s, ptr(out))
    return out


def group_points_grad(grad_out: torch.Tensor, idx: torch.Tensor, n: int) -> torch.Tensor:
    """group_points.cpp:37-60"""
    _chk_contig(grad_out, "grad_out")
    _chk_contig(idx, "idx")
    _chk_float(grad_out, "grad_out")
    _chk_int(idx, "idx")
    if grad_out.is_cuda:
        _chk_cuda(idx, "idx")
    _need_cuda(grad_out)
    b, c = grad_out.size(0), grad_out.size(1)
    m, s = idx.size(1), idx.size(2)
    out = torch.empty((b, c, int(n)), dtype=torch.float32, device=grad_out.device)
    _call("pvn3d_group_points_grad", grad_out.device, ptr(grad_out), ptr(idx), b, c, int(n), m, s, ptr(out))
    return out


def three_nn(unknowns: torch.Tensor, knows: torch.Tensor):
    """interpolate.cpp:14-40 -- returns [dist2 (SQUARED) f32 [B,n,3], idx i32 [B,n,3]]"""
    _chk_contig(unknowns, "unknowns")
    _chk_contig(knows, "knows")
    _chk_float(unknowns, "unknowns")
    _chk_float(knows, "knows")
    if unknowns.is_cuda:
        _chk_cuda(knows, "knows")
    _need_cuda(unknowns)
    b, n = unknowns.size(0), unknowns.size(1)
    m = knows.size(1)
    idx = torch.empty((b, n, 3), dtype=torch.int32, device=unknowns.device)
    dist2 = torch.empty((b, n, 3), dtype=torch.float32, device=unknowns.device)
    _call("pvn3d_three_nn", unknowns.device, ptr(unknowns), ptr(knows), b, n, m, ptr(dist2), ptr(idx))
    return [dist2, idx]


def three_interpolate(points: torch.Tensor, idx: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """interpolate.cpp:42-70 -- points [B,C,M], idx/weight [B,N,3] -> [B,C,N]"""
    _chk_contig(points, "points")
    _chk_contig(idx, "idx")
    _chk_contig(weight, "weight")
    _chk_float(points, "points")
    _chk_int(idx, "idx")
    _chk_float(weight, "weight")
    if points.is_cuda:
        _chk_cuda(idx, "idx")
        _chk_cuda(weight, "weight")
    _need_cuda(points)
    b, c, m = points.shape
    n = idx.size(1)
    out = torch.empty((b, c, n), dtype=torch.float32, device=points.device)
    _call("pvn3d_three_interpolate", points.device, ptr(points), ptr(idx), ptr(weight), b, c, m, n, ptr(out))
    return out


def three_interpolate_grad(grad_out: torch.Tensor, idx: torch.Tensor, weight: torch.Tensor, m: int) -> torch.Tensor:
    """interpolate.cpp:71-97 (intended behaviour, see module docstring)"""
    _chk_contig(grad_out, "grad_out")
    _chk_contig(idx, "idx")
    _chk_contig(weight, "weight")
    _chk_float(grad_out, "grad_out")
    _chk_int(idx, "idx")
    _chk_float(weight, "weight")
    if grad_out.is_cuda:
        _chk_cuda(idx, "idx")
        _chk_cuda(weight, "weight")
    _need_cuda(grad_out)
    b, c, n = grad_out.shape
    out = torch.empty((b, c, int(m)), dtype=torch.float32, device=grad_out.device)
    _call("pvn3d_three_interpolate_grad", grad_out.device, ptr(grad_out), ptr(idx), ptr(weight), b, c, n, int(m), ptr(out))
    return out


# ---- fused forms (not part of the reference module surface; used by pvn3d_b200.pointnet2) --------

def transpose_cn_to_nc(x: torch.Tensor) -> torch.Tensor:
    """[B,C,N] -> [B,N,C] staging copy"""
    _chk_contig(x, "x"); _chk_float(x, "x"); _need_cuda(x)
    b, c, n = x.shape
    out = torch.empty((b, n, c), dtype=torch.float32, device=x.device)
    _call("pvn3d_transpose_cn_to_nc", x.device, ptr(x), b, c, n, ptr(out))
    return out


def transpose_nc_to_cn(x: torch.Tensor) -> torch.Tensor:
    """[B,N,C] -> [B,C,N]"""
    _chk_contig(x, "x"); _chk_float(x, "x"); _need_cuda(x)
    b, n, c = x.shape
    out = torch.empty((b, c, n), dtype=torch.float32, device=x.device)
    _call("pvn3d_transpose_nc_to_cn", x.device, ptr(x), b, n, c, ptr(out))
    return out


def query_and_group(xyz, new_xyz, feat_pm, radius: float, nsample: int, ldf=None, c=None, want_idx=True):
    """QueryAndGroup(radius, nsample, use_xyz=True).forward in one kernel.
    xyz [B,N,3], new_xyz [B,M,3], feat_pm [B,N,ldf] point-major (None -> xyz only).
    Returns (new_features [B,3+C,M,S], idx [B,M,S] or None)."""
    for t, nm in ((xyz, "xyz"), (new_xyz, "new_xyz")):
        _chk_contig(t, nm); _chk_float(t, nm)
    _need_cuda(xyz)
    b, n = xyz.size(0), xyz.size(1)
    m = new_xyz.size(1)
    if feat_pm is not None:
        _chk_contig(feat_pm, "feat_pm"); _chk_float(feat_pm, "feat_pm")
        ldf = feat_pm.size(-1) if ldf is None else int(ldf)
        c = ldf if c is None else int(c)
    else:
        ldf, c = 0, 0
    out = torch.empty((b, 3 + c, m, int(nsample)), dtype=torch.float32, device=xyz.device)
    idx = torch.empty((b, m, int(nsample)), dtype=torch.int32, device=xyz.device) if want_idx else None
    _call("pvn3d_query_and_group", xyz.device, ptr(xyz), ptr(new_xyz), ptr(feat_pm), ldf, b, n, m, c,
          float(radius), int(nsample), ptr(idx), ptr(out))
    return out, idx


def query_and_group2(xyz, new_xyz, feat_pm, radii, nsamples, ldf=None, c=None, want_idx=True, want_out=True):
    """Both scales of an MSG level in one launch.  Returns ([out0, out1], [idx0, idx1]) (None where not wanted)."""
    for t, nm in ((xyz, "xyz"), (new_xyz, "new_xyz")):
        _chk_contig(t, nm); _chk_float(t, nm)
    _need_cuda(xyz)
    b, n = xyz.size(0), xyz.size(1)
    m = new_xyz.size(1)
    if feat_pm is not None and want_out:
        _chk_contig(feat_pm, "feat_pm"); _chk_float(feat_pm, "feat_pm")
        ldf = feat_pm.size(-1) if ldf is None else int(ldf)
        c = ldf if c is None else int(c)
    else:
        ldf, c = (0, 0) if ldf is None else (int(ldf), int(c or 0))
    outs = [torch.empty((b, 3 + c, m, int(ns)), dtype=torch.float32, device=xyz.device) if want_out else None
            for ns in nsamples]
    idxs = [torch.empty((b, m, int(ns)), dtype=torch.int32, device=xyz.device) if want_idx else None for ns in nsamples]
    _call("pvn3d_query_and_group2", xyz.device, ptr(xyz), ptr(new_xyz), ptr(feat_pm) if want_out else 0, ldf, b, n, m, c,
          float(radii[0]), int(nsamples[0]), ptr(idxs[0]), ptr(outs[0]),
          float(radii[1]), int(nsamples[1]), ptr(idxs[1]), ptr(outs[1]))
    return outs, idxs


def ball_query2(new_xyz, xyz, radii, nsamples):
    """ball_query for the two radii of an MSG level in one pass over the cloud -> (idx0, idx1)."""
    _, idxs = query_and_group2(xyz, new_xyz, None, radii, nsamples, want_idx=True, want_out=False)
    return idxs[0], idxs[1]


def three_nn_interpolate(unknown, known, known_feat_pm, out_pm=None, col0=0, want_nn=False):
    """three_nn + inverse-distance weights + three_interpolate on point-major features.
    unknown [B,n,3], known [B,m,3], known_feat_pm [B,m,C] -> out_pm [B,n,ldo] (columns col0..col0+C)."""
    for t, nm in ((unknown, "unknown"), (known, "known"), (known_feat_pm, "known_feat_pm")):
        _chk_contig(t, nm); _chk_float(t, nm)
    _need_cuda(unknown)
    b, n = unknown.size(0), unknown.size(1)
    m, c = known.size(1), known_feat_pm.size(2)
    if out_pm is None:
        out_pm = torch.empty((b, n, c), dtype=torch.float32, device=unknown.device)
    ldo = out_pm.size(2)
    dist2 = torch.empty((b, n, 3), dtype=torch.float32, device=unknown.device) if want_nn else None
    idx = torch.empty((b, n, 3), dtype=torch.int32, device=unknown.device) if want_nn else None
    _call("pvn3d_three_nn_interpolate", unknown.device, ptr(unknown), ptr(known), ptr(known_feat_pm),
          b, n, m, c, ptr(out_pm), ldo, int(col0), ptr(dist2), ptr(idx))
    return out_pm, dist2, idx
