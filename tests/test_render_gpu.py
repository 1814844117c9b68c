"""csrc/render.cu through pvn3d_b200.render.MeshRenderer at LineMOD's 480x640 and K: bit-equal to the numpy
restatement of the raster contract (tests/render_ref.py) on procedural meshes and edge cases, repeatable, graph
capturable, its depth back-projecting onto the posed meshes, the background fill, render and fuse frames through
FrameAugmenter and train_batch, and the refusals."""
import numpy as np
import pytest
import torch

import render_ref as R
from pvn3d_b200 import _lib, augment as A, icp, train_utils as T
from pvn3d_b200._lib import Pvn3dError
from pvn3d_b200.frame_input import FrameInputBuilder
from pvn3d_b200.render import MeshRenderer, pack_meshes

pytestmark = pytest.mark.gpu
H, W, B = 480, 640, 8
N_CLS = 6


def _meshes():
    rng = np.random.default_rng(11)
    sph = R.icosphere(4, 0.06, rng, noise=0.03)                          # 5120 faces
    small = R.icosphere(3, 0.04, rng, noise=0.05)                        # 1280 faces
    bx = R.box(np.array([0.05, 0.04, 0.03]), 12, rng)                    # 1728 faces
    # class 4: one triangle covering the whole frame at 1.5 m, zero-area faces, a triangle with a vertex behind the
    # near plane, and one wholly off the frame
    big = np.array([[-5, -4, 0], [5, -4, 0], [0, 6, 0],
                    [0.1, 0.1, 0], [0.2, 0.2, 0], [0.3, 0.3, 0],                     # collinear
                    [0.1, -0.1, 0.05], [0.1, -0.1, 0.05], [0.2, -0.1, 0.05],         # repeated vertex
                    [-0.3, 0.2, -0.1], [-0.2, 0.2, -1.4995], [-0.3, 0.3, -0.1],       # camera z 5e-4 < z_near
                    [3.0, 0.0, -0.2], [3.5, 0.0, -0.2], [3.2, 0.4, -0.2]], np.float32)  # off the frame
    tri = (big, np.arange(15, dtype=np.int32).reshape(5, 3), rng.integers(0, 256, (15, 3), dtype=np.uint8))
    return {1: sph, 2: bx, 3: sph, 4: tri, 5: small}


def _scene():
    rng = np.random.default_rng(3)
    poses = np.zeros((B, N_CLS, 3, 4))
    present = np.zeros((B, N_CLS), np.uint8)

    def put(f, c, *p):
        poses[f, c] = R.pose(*p)
        present[f, c] = 1
    put(0, 1, 0.2, 0.3, 0.1, (0.0, 0.0, 0.6))                            # render: one object
    put(1, 1, 0.1, 0.2, 0.3, (0.02, 0.0, 0.7))                           # overlapping objects
    put(1, 2, 0.5, -0.4, 0.2, (0.05, 0.02, 0.65))
    put(2, 1, 0.7, 0.1, -0.2, (-0.03, 0.04, 0.5))                        # two classes, same mesh and pose: a tie
    put(2, 3, 0.7, 0.1, -0.2, (-0.03, 0.04, 0.5))
    put(3, 4, 0.0, 0.0, 0.0, (0.0, 0.0, 1.5))                            # full-frame triangle and edge cases
    put(3, 5, 0.3, 0.3, 0.3, (0.0, 0.0, 0.8))
    put(4, 2, 0.2, 0.1, 0.0, (-0.34, 0.1, 0.6))                          # partly off the left edge
    put(4, 5, 0.0, 0.0, 0.0, (2.0, 0.0, 0.6))                            # wholly off the frame
    put(4, 1, 0.0, 0.0, 0.0, (0.1, 0.22, 0.6))                           # partly off the bottom edge
    put(5, 4, 0.05, -0.05, 0.1, (0.01, -0.02, 1.5))
    put(5, 1, 1.0, 2.0, 3.0, (0.05, -0.05, 0.9))
    for f in (6, 7):                                                    # fuse-like scenes
        for c in (1, 2, 5):
            put(f, c, *rng.uniform(-np.pi, np.pi, 3), (rng.uniform(-0.1, 0.1), rng.uniform(-0.08, 0.08),
                                                       rng.uniform(0.5, 0.9)))
    return poses, present


@pytest.fixture(scope="module")
def setup(cuda_dev):
    meshes = _meshes()
    packed = pack_meshes(meshes)
    poses, present = _scene()
    return meshes, packed, poses, present, MeshRenderer(meshes, B, H, W, device=cuda_dev)


def _dev(a, dev, dt=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return t if dt is None else t.to(dt)


def _want(packed, poses, present, background=None):
    vtx, col, faces, vo, fo = packed
    return R.raster(vtx, col, faces, vo, fo, poses, present, R.LM_K, H, W, background=background)


@pytest.mark.parametrize("pose_dtype", [torch.float64, torch.float32])
def test_equals_restatement(setup, cuda_dev, pose_dtype):
    meshes, packed, poses, present, rr = setup
    p = poses.astype(np.float32).astype(np.float64) if pose_dtype == torch.float32 else poses
    rgb, dpt, lab, face = _want(packed, p, present)
    g_rgb, g_dpt, g_lab = rr.render(_dev(poses, cuda_dev, pose_dtype), _dev(present, cuda_dev),
                                    _dev(R.LM_K, cuda_dev))
    g_rgb, g_dpt, g_lab = g_rgb.cpu().numpy(), g_dpt.cpu().numpy(), g_lab.cpu().numpy()
    assert np.array_equal(g_lab, lab), [int((g_lab[f] != lab[f]).sum()) for f in range(B)]
    assert np.array_equal(g_dpt.view(np.uint32), dpt.view(np.uint32))
    assert np.array_equal(g_rgb, rgb)
    # the scene exercises what it claims to
    assert (lab[0] == 1).sum() > 5000 and set(np.unique(lab[1])) == {0, 1, 2}
    assert set(np.unique(lab[2])) == {0, 1}                              # class 1 wins every tie with class 3
    assert (lab[3] > 0).all() and (lab[3] == 5).sum() > 1000            # the whole frame is covered
    assert (lab[4, :, 0] == 2).any() and (lab[4, -1] == 1).any() and not (lab[4] == 5).any()
    assert (face[3] == -1).sum() == 0 and set(np.unique(face[3][lab[3] == 4])) == {int(packed[4][4])}


def test_repeat_and_graph(setup, cuda_dev):
    meshes, packed, poses, present, rr = setup
    K = _dev(R.LM_K, cuda_dev)
    pr = _dev(present, cuda_dev)
    ps = _dev(poses, cuda_dev)
    first = [t.clone() for t in rr.render(ps, pr, K)]
    again = rr.render(ps, pr, K)
    assert all(torch.equal(a, b) for a, b in zip(first, again))
    torch.cuda.synchronize()
    s = torch.cuda.Stream(cuda_dev)
    s.wait_stream(torch.cuda.current_stream(cuda_dev))
    with torch.cuda.stream(s):
        rr.render(ps, pr, K)                                             # warm on the capture stream
    torch.cuda.current_stream(cuda_dev).wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = rr.render(ps, pr, K)
    moved = poses.copy()
    moved[..., 3] += np.array([0.01, -0.02, 0.05])
    moved[:, :, :3, :3] = np.einsum("ij,bcjk->bcik", R.pose(0.1, 0.2, 0.0, (0, 0, 0))[:, :3], poses[:, :, :3, :3])
    ps.copy_(_dev(moved, cuda_dev))                                      # the pose table changes in place
    g.replay()
    torch.cuda.synchronize()
    replayed = [t.clone() for t in out]
    eager = rr.render(_dev(moved, cuda_dev), pr, K)
    assert all(torch.equal(a, b) for a, b in zip(replayed, eager))
    assert not torch.equal(replayed[2], first[2])
    want = _want(packed, moved, present)
    assert np.array_equal(replayed[2].cpu().numpy(), want[2])


def _bound(z):
    # the displaced triangle: <= 1/512 px per axis of vertex shift, plus float32 depth and back-projection rounding
    return z * (np.sqrt(2) / (512 * min(R.LM_K[0, 0], R.LM_K[1, 1])) + 2.0 ** -20)


def test_depth_backprojects_onto_meshes(setup, cuda_dev):
    meshes, packed, poses, present, rr = setup
    _, dpt, lab = rr.render(_dev(poses, cuda_dev), _dev(present, cuda_dev), _dev(R.LM_K, cuda_dev))
    K32 = _dev(np.repeat(R.LM_K[None], B, 0), cuda_dev, torch.float32)
    cloud, valid = icp.depth_to_cloud(dpt, K32, torch.ones(B, device=cuda_dev))
    cloud, lab = cloud.cpu().numpy().reshape(B, H * W, 3), lab.cpu().numpy().reshape(B, -1)
    face = _want(packed, poses, present)[3].reshape(B, -1)
    vtx, _, faces, _, fo = packed
    cls_f = np.repeat(np.arange(N_CLS), np.diff(fo))
    n = 0
    for f in range(B):
        sel = np.nonzero(lab[f])[0]
        fid = face[f, sel]
        dist = R.plane_distance(cloud[f, sel].astype(np.float64), vtx, faces, fid, poses[f, cls_f[fid]])
        z = cloud[f, sel, 2].astype(np.float64)
        assert np.all(dist <= _bound(z)), (f, float((dist / _bound(z)).max()))
        n += sel.size
    assert n > 300000


def test_background_fill(setup, cuda_dev):
    meshes, packed, poses, present, rr = setup
    rng = np.random.default_rng(4)
    back_rgb = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
    back_dpt = rng.uniform(0.3, 2.0, (B, H, W)).astype(np.float32)
    ps, pr, K = _dev(poses, cuda_dev), _dev(present, cuda_dev), _dev(R.LM_K, cuda_dev)
    plain = [t.cpu().numpy() for t in rr.render(ps, pr, K)]
    fused = [t.cpu().numpy() for t in rr.render(ps, pr, K, background=(_dev(back_rgb, cuda_dev),
                                                                      _dev(back_dpt, cuda_dev)))]
    cov = plain[2] > 0
    assert np.array_equal(fused[2], plain[2])
    assert np.array_equal(fused[0][cov], plain[0][cov]) and np.array_equal(fused[1][cov], plain[1][cov])
    assert np.array_equal(fused[0][~cov], back_rgb[~cov]) and np.array_equal(fused[1][~cov], back_dpt[~cov])
    want = _want(packed, poses, present, background=(back_rgb, back_dpt))
    assert all(np.array_equal(a, b) for a, b in zip(fused, want[:3]))


def test_render_and_fuse_frames_train(setup, cuda_dev):
    meshes, packed, poses, present, _ = setup
    obj = 1
    b, n = 2, 12288
    rr = MeshRenderer(meshes, b, H, W, device=cuda_dev)
    rng = np.random.default_rng(8)
    real_rgb = rng.integers(0, 256, (b, H, W, 3), dtype=np.uint8)
    real_dpt = rng.uniform(0.9, 1.4, (b, H, W)).astype(np.float32)      # metres: cam_scale = 1
    fp = np.zeros((b, N_CLS, 3, 4))
    fpr = np.zeros((b, N_CLS), np.uint8)
    fp[0, obj], fpr[0, obj] = R.pose(0.3, -0.2, 0.4, (0.01, -0.02, 0.65)), 1              # render frame
    fp[1, obj], fpr[1, obj] = R.pose(-0.5, 0.6, 0.1, (-0.04, 0.02, 0.7)), 1               # fuse frame: obj and two
    fp[1, 2], fpr[1, 2] = R.pose(0.2, 0.2, 0.2, (0.08, 0.05, 0.75)), 1                   # other objects
    fp[1, 5], fpr[1, 5] = R.pose(0.1, 0.9, 0.2, (-0.1, -0.06, 0.6)), 1
    K = _dev(R.LM_K, cuda_dev)
    rgb0, dpt0, lab0 = [t.clone() for t in rr.render(_dev(fp[:1], cuda_dev), _dev(fpr[:1], cuda_dev), K)]
    rgb1, dpt1, lab1 = rr.render(_dev(fp[1:], cuda_dev), _dev(fpr[1:], cuda_dev), K,
                                 background=(_dev(real_rgb[1:], cuda_dev), _dev(real_dpt[1:], cuda_dev)))
    rgb = torch.cat([rgb0, rgb1])
    dpt = torch.cat([dpt0, dpt1])
    # get_item's masks: a render frame's labels > 0, a fuse frame's labels == cls_id
    label_image = torch.stack([(lab0[0] > 0), (lab1[0] == obj)]).to(torch.uint8)
    aug = A.FrameAugmenter(b, "linemod", H, W, device=cuda_dev)
    back_lab = torch.zeros((b, H, W), dtype=torch.uint8, device=cuda_dev)
    params = aug.draw(5, ["render", "fuse"])
    rgb_a, dpt_a = aug.apply(rgb, dpt, label_image, _dev(real_rgb, cuda_dev), back_lab, _dev(real_dpt, cuda_dev),
                             params)
    builder = FrameInputBuilder(b, n, device=cuda_dev)
    targets = T.TrainTargets.linemod(obj, device=cuda_dev)
    K32 = _dev(np.repeat(R.LM_K[None], b, 0), cuda_dev, torch.float32)
    ids = torch.ones((b, 1), dtype=torch.int32, device=cuda_dev)
    rts = _dev(fp[:, obj][:, None], cuda_dev)
    out = T.train_batch(builder, targets, dpt_a, K32, torch.ones(b, device=cuda_dev), rgb_a, label_image, ids, rts,
                        seed=3)
    assert out[-1].tolist() == [1, 1]
    pcld, choose, labels = out[1].cpu().numpy(), out[3].cpu().numpy()[:, 0], out[8].cpu().numpy()
    vtx, _, faces, _, fo = packed
    for f, (p, pr) in enumerate(((fp[:1], fpr[:1]), (fp[1:], fpr[1:]))):
        face = R.raster(*packed, p, pr, R.LM_K, H, W)[3][0].reshape(-1)
        sel = np.nonzero(labels[f] == 1)[0]
        assert sel.size > 100
        fid = face[choose[f, sel]]
        assert (fid >= fo[obj]).all() and (fid < fo[obj + 1]).all()      # every object point is the object's pixel
        dist = R.plane_distance(pcld[f, sel].astype(np.float64), vtx, faces, fid, np.repeat(fp[f, obj][None], sel.size, 0))
        assert np.all(dist <= _bound(pcld[f, sel, 2].astype(np.float64))), f


def test_refusals(setup, cuda_dev):
    meshes, packed, poses, present, rr = setup
    ps, pr, K = _dev(poses, cuda_dev), _dev(present, cuda_dev), _dev(R.LM_K, cuda_dev)
    bad = [
        dict(poses=ps[:, :4]),                                          # class count
        dict(poses=ps.to(torch.float16)),
        dict(poses=torch.cat([ps, ps])),                                # more frames than the batch
        dict(poses=ps.cpu()),
        dict(present=pr[:, :3]),
        dict(present=pr.float()),
        dict(K=K[:2]),
        dict(K=K.to(torch.int32)),
        dict(background=(torch.zeros((B, H, W, 3), dtype=torch.uint8, device=cuda_dev),)),
        dict(background=(torch.zeros((B, H, W, 3), dtype=torch.uint8, device=cuda_dev),
                         torch.zeros((B, H, W), dtype=torch.float64, device=cuda_dev))),
        dict(background=(torch.zeros((B, H, W - 1, 3), dtype=torch.uint8, device=cuda_dev),
                         torch.zeros((B, H, W - 1), dtype=torch.float32, device=cuda_dev))),
    ]
    for kw in bad:
        args = dict(poses=ps, present=pr, K=K)
        args.update(kw)
        with pytest.raises(ValueError):
            rr.render(**args)
    for kw in (dict(height=4097), dict(width=0), dict(batch=0), dict(z_near=0.0), dict(z_near=float("nan"))):
        a = dict(batch=1, height=H, width=W)
        a.update(kw)
        with pytest.raises(ValueError):
            MeshRenderer(meshes, device=cuda_dev, **a)
    with pytest.raises(RuntimeError):
        MeshRenderer(meshes, 1, H, W, device="cpu")
    lib = _lib.load()
    assert lib.pvn3d_render_workspace_bytes(1, 4097, 640, 10, 10) == 0
    assert lib.pvn3d_render_workspace_bytes(0, 480, 640, 10, 10) == 0
    assert lib.pvn3d_render_workspace_bytes(65536, 1, 1, 1, 1) == 0
    # the C ABI's own checks: null pointers, z_near, one background buffer without the other, a short workspace
    t = [rr.vtx, rr.colors, rr.faces, rr.vtx_off, rr.face_off]
    ptrs = [x.data_ptr() for x in t]
    kk = K.to(torch.float64).expand(1, 3, 3).contiguous()
    stream = torch.cuda.current_stream(cuda_dev).cuda_stream

    def call(z_near=1e-3, back=(0, 0), ws=None, vtx=None, n_cls=N_CLS, h=H):
        ws_ptr, ws_bytes = (rr._ws[1], rr._ws_bytes) if ws is None else ws
        return lib.pvn3d_render_meshes(ptrs[0] if vtx is None else vtx, *ptrs[1:], n_cls, rr.n_vtx, rr.n_faces,
                                       ps.data_ptr(), 1, pr.data_ptr(), kk.data_ptr(), 1, h, W, z_near, back[0],
                                       back[1], rr.rgb.data_ptr(), rr.depth.data_ptr(), rr.labels.data_ptr(), ws_ptr,
                                       ws_bytes, stream)
    assert call() == 0
    assert call(vtx=0) == -1
    assert call(z_near=0.0) == -1 and call(z_near=float("inf")) == -1
    assert call(back=(rr.rgb.data_ptr(), 0)) == -1
    assert call(ws=(rr._ws[1], 1024)) == -4
    assert call(ws=(rr._ws[1] + 8, rr._ws_bytes)) == -1
    assert call(n_cls=257) == -2 and call(h=4097) == -2 and call(n_cls=1) == -1
    with pytest.raises(Pvn3dError):
        _lib.check(call(vtx=0), "pvn3d_render_meshes")
    torch.cuda.synchronize()
