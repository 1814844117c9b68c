"""csrc/render.cu at its edges (tests/render_edge_cases.py): rgb, depth bits and labels equal the numpy restatement
of the raster contract bit for bit, frame by frame, at the benchmark's shape and on past the scan's block and pass
boundaries, the guard band and near plane, per-frame K, odd frame sizes, 256 classes, non-finite and mirrored poses
and 11,500 contending faces; and a 4096x4096 frame of more than 2^32 fragments equals its analytic result.  What
each case reaches is shown on the host (test_render_edges_host.py)."""
import numpy as np
import pytest
import torch

import render_edge_cases as E
import render_ref as R
from pvn3d_b200 import _lib
from pvn3d_b200.render import MeshRenderer

pytestmark = pytest.mark.gpu


def _dev(a, dev, dt=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return t if dt is None else t.to(dt)


def _render(rr, case, dev, frames=slice(None), pose_dtype=torch.float64, K=None, background=None):
    K = case.K if K is None else K
    kk = K if K.ndim == 2 else K[frames]
    out = rr.render(_dev(case.poses[frames], dev, pose_dtype), _dev(case.present[frames], dev), _dev(kk, dev),
                    background=None if background is None else tuple(_dev(x, dev) for x in background))
    return [t.cpu().numpy() for t in out]


def _assert_equal(got, want, name):
    for f in range(want[2].shape[0]):
        assert np.array_equal(got[2][f], want[2][f]), (name, f, "labels", int((got[2][f] != want[2][f]).sum()))
        assert np.array_equal(got[1][f].view(np.uint32), want[1][f].view(np.uint32)), (name, f, "depth")
        assert np.array_equal(got[0][f], want[0][f]), (name, f, "rgb")


def _check(case, dev, **kw):
    rr = MeshRenderer(case.meshes, case.b, case.h, case.w, case.z_near, device=dev)
    got = _render(rr, case, dev, **kw)
    f32 = kw.get("pose_dtype") == torch.float32
    _assert_equal(got, case.want(poses=case.poses.astype(np.float32).astype(np.float64) if f32 else None), case.name)
    return rr, got


def test_bench_shape(cuda_dev):
    case = E.bench()
    rr, got = _check(case, cuda_dev)
    assert (got[2][:16] > 0).sum() > 0 and len(np.unique(got[2][16:])) == 5
    # fewer frames than the batch after the full one, with a background: the last 8 (fuse) frames
    rng = np.random.default_rng(22)
    sub = slice(24, 32)
    back = (rng.integers(0, 256, (8, case.h, case.w, 3), dtype=np.uint8),
            rng.uniform(0.3, 2.0, (8, case.h, case.w)).astype(np.float32))
    got = _render(rr, case, cuda_dev, frames=sub, background=back)
    want = R.raster(*case.packed, case.poses[sub], case.present[sub], case.K, case.h, case.w, background=back)
    _assert_equal(got, want, "bench, frames 24-31 over a background")


@pytest.mark.parametrize("variant", sorted(E.SCAN_VARIANTS))
def test_scan_boundaries(variant, cuda_dev):
    _check(E.scan(variant), cuda_dev)


def test_over_2e32_fragments(cuda_dev):
    case, rgb, dpt, lab = E.over_2e32()
    rr = MeshRenderer(case.meshes, 1, E.BIG, E.BIG, device=cuda_dev)
    ps, pr, K = _dev(case.poses, cuda_dev), _dev(case.present, cuda_dev), _dev(case.K, cuda_dev)
    first = None
    for _ in range(3):
        out = rr.render(ps, pr, K)
        torch.cuda.synchronize()
        if first is None:
            first = [t.clone() for t in out]
            g = [t.cpu().numpy() for t in out]
            assert np.array_equal(g[2], lab), int((g[2] != lab).sum())
            assert np.array_equal(g[1].view(np.uint32), dpt.view(np.uint32))
            assert np.array_equal(g[0], rgb)
        else:
            assert all(torch.equal(a, b) for a, b in zip(first, out))


def test_guard_and_near(cuda_dev):
    _check(E.guard(), cuda_dev)


@pytest.mark.parametrize("k_form", ["float32 [B,3,3]", "float64 [3,3]"])
def test_per_frame_k(k_form, cuda_dev):
    case = E.per_frame_k()
    rr = MeshRenderer(case.meshes, case.b, case.h, case.w, device=cuda_dev)
    if k_form == "float32 [B,3,3]":
        k32 = case.K.astype(np.float32)
        got = _render(rr, case, cuda_dev, K=k32)
        want = case.want(K=k32.astype(np.float64))
        assert all(got[2][f].any() for f in range(case.b))             # every K shows its frame's objects
    else:
        got = _render(rr, case, cuda_dev, K=case.K[4])                  # skew and row 2 set, not read
        want = case.want(K=case.K[4])
    _assert_equal(got, want, f"per-frame K, {k_form}")


@pytest.mark.parametrize("size", E.SIZES, ids=[f"{h}x{w}" for h, w in E.SIZES])
def test_frame_sizes(size, cuda_dev):
    _, got = _check(E.frame_size(*size), cuda_dev)
    assert got[2].any()


def test_tiny_frames(cuda_dev):
    _, got = _check(E.tiny_frames(), cuda_dev)
    assert (got[2] > 0).any(axis=(1, 2)).sum() > 500


@pytest.mark.parametrize("form", ["dict", "list"])
def test_class_layouts(form, cuda_dev):
    case = E.classes(as_list=form == "list")
    _, got = _check(case, cuda_dev)
    assert (got[2][1] == 255).any()


def test_foreign_faces_through_c_abi(cuda_dev):
    case = E.foreign_faces()
    lib = _lib.load()
    vtx, col, faces, vo, fo = (_dev(a, cuda_dev) for a in case.packed)
    b, h, w = case.b, case.h, case.w
    n_cls, n_vtx, n_faces = vo.numel() - 1, vtx.shape[0], faces.shape[0]
    ps, pr = _dev(case.poses, cuda_dev), _dev(case.present, cuda_dev)
    kk = _dev(np.broadcast_to(case.K, (b, 3, 3)), cuda_dev)
    ws_bytes = lib.pvn3d_render_workspace_bytes(b, h, w, n_vtx, n_faces)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=cuda_dev)     # the caching allocator aligns to 512 B
    rgb = torch.empty((b, h, w, 3), dtype=torch.uint8, device=cuda_dev)
    depth = torch.empty((b, h, w), dtype=torch.float32, device=cuda_dev)
    labels = torch.empty((b, h, w), dtype=torch.uint8, device=cuda_dev)
    rc = lib.pvn3d_render_meshes(vtx.data_ptr(), col.data_ptr(), faces.data_ptr(), vo.data_ptr(), fo.data_ptr(),
                                 n_cls, n_vtx, n_faces, ps.data_ptr(), 1, pr.data_ptr(), kk.data_ptr(), b, h, w, 1e-3,
                                 0, 0, rgb.data_ptr(), depth.data_ptr(), labels.data_ptr(), ws.data_ptr(), ws_bytes,
                                 torch.cuda.current_stream(cuda_dev).cuda_stream)
    assert rc == 0                                                      # PVN3D_OK
    torch.cuda.synchronize()
    _assert_equal([rgb.cpu().numpy(), depth.cpu().numpy(), labels.cpu().numpy()], case.want(), case.name)


@pytest.mark.parametrize("pose_dtype", [torch.float64, torch.float32])
def test_poses(pose_dtype, cuda_dev):
    _check(E.poses(), cuda_dev, pose_dtype=pose_dtype)


def test_contention(cuda_dev):
    case = E.contention()
    want = case.want()
    rr = MeshRenderer(case.meshes, 1, case.h, case.w, device=cuda_dev)
    for _ in range(3):
        _assert_equal(_render(rr, case, cuda_dev), want, case.name)
