"""The pose overlay on the GPU (csrc/vis.cu through pvn3d_b200.vis_utils) against the goldens recorded from the
reference (tests/golden/vis_cases.npz), bit for bit: PoseOverlay.draw on every overlay case (float64 and float32
poses), the draw_p2ds drop-in on every point case, a batch against the per-frame loop, repeat calls, sync-debug mode,
CUDA graph capture, the refusals, and compat's patched Basic_Utils.draw_p2ds on the staged reference."""
import os

import numpy as np
import pytest
import torch

import vis_ref as V
from helpers import load_reference_python
from pvn3d_b200 import compat, vis_utils
from pvn3d_b200._lib import Pvn3dError
from pvn3d_b200.vis_utils import PoseOverlay
from test_vis_host import frame_images, overlay_case

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def g():
    return dict(np.load(os.path.join(ROOT, "tests", "golden", "vis_cases.npz")))


def _inputs(c, dev, pose_dtype=torch.float64):
    b = len(c.seeds)
    img = torch.from_numpy(np.stack([V.background(int(s), c.h, c.w) for s in c.seeds])).to(dev)
    colors = torch.from_numpy(np.stack([V.cv_color(x) for x in c.colors])).to(dev)
    return (img, torch.from_numpy(c.poses).to(dev, pose_dtype), torch.from_numpy(c.present).to(dev),
            torch.from_numpy(c.order).to(dev).reshape(b, -1, 1), torch.from_numpy(c.K).to(dev), colors)


def test_overlay_equals_goldens(g, cuda_dev):
    for i in range(int(g["n_overlay"])):
        c = overlay_case(g, i)
        want = np.stack(frame_images(g, c.k, c.h, c.w))
        ov = PoseOverlay(c.meshes, cuda_dev)
        for dt in (torch.float64, torch.float32):           # the recorded poses are float32-representable
            img, poses, present, order, K, colors = _inputs(c, cuda_dev, dt)
            out = ov.draw(img, poses, present, order, K, colors, radius=c.r, cam_scale=c.cam_scale)
            assert out is img
            got = img.cpu().numpy()
            assert np.array_equal(got, want), (c.name, dt, int((got != want).any(-1).sum()))
            assert all(V.sha(got[f]) == g[c.k + "sha"][f].tobytes() for f in range(len(got)))


def test_draw_p2ds_equals_goldens(g, cuda_dev):
    for i in range(int(g["n_p2ds"])):
        k = f"dp{i}_"
        h, w = (int(x) for x in g[k + "hw"])
        (want,) = frame_images(g, k, h, w)
        for dt in (np.int32, np.int64):
            img = V.background(int(g[k + "seeds"][0]), h, w)
            p = g[k + "p2ds_in"].astype(dt)
            out = vis_utils.draw_p2ds(img, p, r=int(g[k + "r"]), color=tuple(g[k + "color"]))
            assert out is img                                   # drawn in place, the same array returned
            assert np.array_equal(img, want), (k, dt)
            assert p.dtype == dt and np.array_equal(p, g[k + "p2ds_out"]), (k, dt)   # clipped in place


def test_batch_equals_per_frame_loop(g, cuda_dev):
    # four frames: the two YCB frames, then the same poses drawn in reversed slot order and with a second K
    c = overlay_case(g, 0)
    img, poses, present, order, K, colors = _inputs(c, cuda_dev)
    order = order.reshape(2, -1)
    k2 = K[0].clone()
    k2[0, 2] += 17.0
    img4 = torch.cat([img, img.flip(1).contiguous()])
    poses4, present4 = torch.cat([poses, poses]), torch.cat([present, present])
    order4 = torch.cat([order, order.flip(1)])
    K4 = torch.stack([K[0], K[1], k2, K[0]])
    ov = PoseOverlay(c.meshes, cuda_dev)
    batch = ov.draw(img4.clone(), poses4, present4, order4, K4, colors).cpu()
    for f in range(4):
        one = ov.draw(img4[f:f + 1].clone(), poses4[f:f + 1], present4[f:f + 1], order4[f:f + 1], K4[f:f + 1],
                      colors).cpu()
        assert torch.equal(one[0], batch[f]), f
    # and the numpy restatement of the reversed-order frame (a different slot wins where discs meet)
    meshes = c.meshes
    ref, _ = V.overlay_frame(img4[2].cpu().numpy(), meshes, c.poses[0], c.present[0], order4[2].cpu().numpy(),
                             k2.cpu().numpy(), c.colors, 1, 1.0)
    assert np.array_equal(batch[2].numpy(), ref)


def test_repeat_calls_give_the_same_bits(g, cuda_dev):
    c = overlay_case(g, 6)
    ov = PoseOverlay(c.meshes, cuda_dev)
    img, poses, present, order, K, colors = _inputs(c, cuda_dev)
    outs = [ov.draw(img.clone(), poses, present, order, K, colors, radius=c.r).cpu() for _ in range(3)]
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


def test_no_host_sync_and_graph_capture(g, cuda_dev):
    c = overlay_case(g, 0)
    want = torch.from_numpy(np.stack(frame_images(g, c.k, c.h, c.w)))
    ov = PoseOverlay(c.meshes, cuda_dev)
    img, poses, present, order, K, colors = _inputs(c, cuda_dev)
    bg = img.clone()
    ov.draw(img, poses, present, order, K, colors)               # warm-up: the workspace exists
    img.copy_(bg)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        ov.draw(img, poses, present, order, K, colors)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(img.cpu(), want)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        img.copy_(bg)
        with torch.cuda.graph(graph, stream=s):
            img.copy_(bg)
            ov.draw(img, poses, present, order, K, colors)
    torch.cuda.current_stream().wait_stream(s)
    img.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(img.cpu(), want)
    poses.zero_()                 # a replay reads the captured tensors' new values: every point now projects to (0, 0)
    img.zero_()
    graph.replay()
    torch.cuda.synchronize()
    for f in range(2):
        ref, _ = V.overlay_frame(bg[f].cpu().numpy(), c.meshes, np.zeros_like(c.poses[f]), c.present[f], c.order[f],
                                 c.K[f], c.colors)
        assert np.array_equal(img[f].cpu().numpy(), ref), f


def test_refusals(g, cuda_dev):
    c = overlay_case(g, 1)
    ov = PoseOverlay(c.meshes, cuda_dev)
    img, poses, present, order, K, colors = _inputs(c, cuda_dev)
    with pytest.raises(ValueError):
        ov.draw(img.float(), poses, present, order, K, colors)                       # dtype
    with pytest.raises(ValueError):
        ov.draw(img.permute(0, 2, 1, 3), poses, present, order, K, colors)           # layout
    with pytest.raises(ValueError):
        ov.draw(img.cpu(), poses, present, order, K, colors)                         # not on the device
    with pytest.raises(ValueError):
        ov.draw(img, poses.half(), present, order, K, colors)
    with pytest.raises(ValueError):
        ov.draw(img, poses, present, order.float(), K, colors)
    with pytest.raises(ValueError):
        ov.draw(img, poses, present, order, K, colors.int())
    with pytest.raises(ValueError):
        ov.draw(img, poses, present, order, K, colors, radius=-1)                    # r < 0
    with pytest.raises(ValueError):                                                  # a class without a mesh
        ov.draw(img, torch.cat([poses, poses[:, 1:]], 1), torch.cat([present, present[:, 1:]], 1), order, K,
                torch.cat([colors, colors[1:]]))
    with pytest.raises(ValueError):
        PoseOverlay({1: c.meshes[1], 3: c.meshes[1]}, cuda_dev)                      # class 2 has no mesh
    with pytest.raises(RuntimeError):
        PoseOverlay(c.meshes, "cpu")
    with pytest.raises(ValueError):
        vis_utils.draw_p2ds(np.zeros((4, 5, 3), np.uint8), np.zeros((2, 2), np.int32), r=-2)
    # the C ABI refuses what the wrapper would not pass
    from pvn3d_b200 import _lib

    lib = _lib.load()
    ws = torch.zeros(lib.pvn3d_vis_workspace_bytes(1, c.h, c.w), dtype=torch.uint8, device=cuda_dev)
    p = torch.zeros((3, 2), dtype=torch.int32, device=cuda_dev)
    with pytest.raises(Pvn3dError, match="invalid argument"):
        _lib.check(lib.pvn3d_vis_draw_p2ds(img.data_ptr(), c.h, c.w, p.data_ptr(), 3, -1, 0, ws.data_ptr(), ws.numel(),
                                           None), "pvn3d_vis_draw_p2ds")
    with pytest.raises(Pvn3dError, match="workspace too small"):
        _lib.check(lib.pvn3d_vis_draw_p2ds(img.data_ptr(), c.h, c.w, p.data_ptr(), 3, 1, 0, ws.data_ptr(),
                                           ws.numel() - 4, None), "pvn3d_vis_draw_p2ds")
    # nothing was drawn by any refused call
    assert torch.equal(img.cpu(), torch.from_numpy(V.background(int(c.seeds[0]), c.h, c.w))[None])


def test_patched_draw_p2ds_equals_reference_on_staged_reference(g, cuda_dev):
    ref = load_reference_python()
    if ref is None:
        pytest.skip("reference Python not staged under oracle/_ref/py")
    cls = ref.basic_utils.Basic_Utils
    orig = cls.draw_p2ds
    import types

    bu = cls(types.SimpleNamespace(dataset_name="linemod"))
    try:
        compat.patch_vis_modules()
        assert cls.draw_p2ds._pvn3d_b200_orig is orig
        for i in range(int(g["n_p2ds"])):
            k = f"dp{i}_"
            h, w = (int(x) for x in g[k + "hw"])
            seed, r, color = int(g[k + "seeds"][0]), int(g[k + "r"]), tuple(float(v) for v in g[k + "color"])
            a_img, a_p = V.background(seed, h, w), g[k + "p2ds_in"].copy()
            b_img, b_p = V.background(seed, h, w), g[k + "p2ds_in"].copy()
            a = orig(bu, a_img, a_p, r=r, color=color)
            b = bu.draw_p2ds(b_img, b_p, r=r, color=color)
            assert b is b_img and np.array_equal(a, b) and np.array_equal(a_p, b_p), k
        # demo.py's own composition on the LineMOD case, through the patched instance
        c = overlay_case(g, 1)
        img = V.background(int(c.seeds[0]), c.h, c.w)
        mesh = np.dot(c.meshes[1], c.poses[0, 1][:, :3].T) + c.poses[0, 1][:, 3]
        p2ds = bu.project_p3d(mesh, 1.0, c.K[0])
        img = bu.draw_p2ds(img, p2ds, color=tuple(c.colors[1]))
        assert np.array_equal(img, frame_images(g, c.k, c.h, c.w)[0])
        # a call the GPU path does not take (points as a list) runs the reference's method
        a_img, b_img = np.zeros((8, 8, 3), np.uint8), np.zeros((8, 8, 3), np.uint8)
        assert np.array_equal(bu.draw_p2ds(a_img, [[3, 4], [9, -2]], r=2), orig(bu, b_img, [[3, 4], [9, -2]], r=2))
    finally:
        cls.draw_p2ds = orig
