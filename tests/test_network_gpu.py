"""The whole PVN3D network forward on the fused engines (pvn3d_b200.network.FusedPVN3D) and the PVN3D.forward patch.

  * pvn3d_gather_pixel_rows and pvn3d_mlp_fp_fact2_rows against the tensors they replace, bit for bit;
  * FusedPVN3D against the hand composition FusedHeads(gathered rgb_emb, FusedPointnet2MSG(pointcloud)), bit for bit;
  * FusedPVN3D against the reference's PVN3D.forward (tests/golden/network_ref.npz, tests/golden/make_golden_network.py)
    within the tolerance of tests/test_heads_gpu.py;
  * compat.patch_pvn3d_forward: which calls take the fused path, and the engine cache.
"""
import os

import numpy as np
import pytest
import torch

from pvn3d_b200 import _lib, compat, eval_utils, fixtures, mlp, network, testing
from pvn3d_b200.eval_utils import FramePoseSolver
from pvn3d_b200.heads import FusedHeads

from network_cases import NETWORK_CASES, network_inputs, network_model, network_points

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fp32_reference():
    """the unfused paths below run in fp32, as the golden was recorded"""
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _gather_ref(emb, choose):
    b, c = emb.shape[:2]
    g = torch.gather(emb.reshape(b, c, -1), 2, choose.repeat(1, c, 1))
    return mlp.tf32_round(g.transpose(1, 2).contiguous()).reshape(-1, c)


def _sentinel_table(rows, cols, dev):
    return torch.full((rows, cols), -7.25, dtype=torch.float32, device=dev)


@pytest.mark.parametrize("b,c,hw,n", [(2, 128, 120 * 160, 4096), (3, 32, 500, 1000)])
def test_gather_pixel_rows_bit_exact(cuda_dev, b, c, hw, n):
    g = torch.Generator().manual_seed(c + n)
    emb = torch.randn(b, c, hw, generator=g).to(cuda_dev)
    choose = testing.sample_choose(b, n, hw, seed=n)
    choose[0, 0, :3] = torch.tensor([0, hw - 1, hw - 1])      # both ends of the image, a duplicate
    choose[-1, 0, -1] = 0
    choose = choose.to(cuda_dev)
    col0, ldo = 128, 1280
    out = _sentinel_table(b * n, ldo, cuda_dev)
    network.gather_pixel_rows(emb, choose, out, col0=col0)
    want = _gather_ref(emb, choose)
    assert torch.equal(out[:, col0:col0 + c], want)
    assert bool((out[:, :col0] == -7.25).all()) and bool((out[:, col0 + c:] == -7.25).all())


def test_gather_out_of_range_index_gives_a_nan_row(cuda_dev):
    b, c, hw, n = 2, 128, 4000, 1000
    emb = torch.randn(b, c, hw, generator=torch.Generator().manual_seed(1)).to(cuda_dev)
    choose = testing.sample_choose(b, n, hw, seed=3)
    bad = [(0, 5), (1, 999)]
    choose[0, 0, 5], choose[1, 0, 999] = hw, -1
    out = _sentinel_table(b * n, 256, cuda_dev)
    network.gather_pixel_rows(emb, choose.to(cuda_dev), out, col0=0)
    bad_rows = torch.tensor([f * n + p for f, p in bad])
    good = torch.ones(b * n, dtype=torch.bool)
    good[bad_rows] = False
    good = good.to(cuda_dev)
    assert bool(torch.isnan(out[bad_rows.to(cuda_dev), :c]).all())
    assert not bool(torch.isnan(out[good]).any())
    safe = choose.clone()
    safe[0, 0, 5] = safe[1, 0, 999] = 0
    assert torch.equal(out[good, :c], _gather_ref(emb, safe.to(cuda_dev))[good])
    assert bool((out[:, c:] == -7.25).all())


def _fp1_module(dev, b, n, m, seed):
    g = torch.Generator().manual_seed(seed)
    xyz = (torch.rand(b, n, 3, generator=g) * 2 - 1).to(dev)
    feat = torch.randn(b * n, 6, generator=g).to(dev)
    p = (torch.randn(b * m, 128, generator=g) * 0.5).to(dev)
    nn_idx = torch.randint(0, m, (b, n, 3), generator=g, dtype=torch.int32).to(dev)
    w = torch.rand(b, n, 3, generator=g) + 0.05
    nn_w = (w / w.sum(-1, keepdim=True)).to(dev)
    ws = torch.randn(128, 9, generator=g) / 3
    ls = mlp.PackedLayer(torch.cat([ws, ws[:, 6:]], dim=1), torch.randn(128, generator=g) * 0.1)
    l2 = mlp.PackedLayer(torch.randn(128, 128, generator=g) * 128 ** -0.5, torch.randn(128, generator=g) * 0.1, ls.n_pad)
    ls.w, ls.bias, l2.w, l2.bias = (t.to(dev) for t in (ls.w, ls.bias, l2.w, l2.bias))
    table = mlp.sa_factor_table(xyz, feat.data_ptr(), 6, 6, ls.k_pad)
    return p, table, nn_idx, nn_w, ls, l2


@pytest.mark.parametrize("b,n,m", [(2, 12288, 2048), (3, 1000, 333)])   # 1000 points: 64-row tiles straddle frames
def test_fp1_rows_bit_exact(cuda_dev, b, n, m):
    p, table, nn_idx, nn_w, ls, l2 = _fp1_module(cuda_dev, b, n, m, seed=n)
    cn = mlp.mlp_fp_fact2(p, table, nn_idx, nn_w, m, ls, l2)                     # [b, 128, n]
    want = mlp.tf32_round(cn.transpose(1, 2).contiguous()).reshape(b * n, 128)
    out = _sentinel_table(b * n, 1280, cuda_dev)
    mlp.mlp_fp_fact2_rows(p, table, nn_idx, nn_w, m, ls, l2, out, 128)
    assert torch.equal(out[:, 128:256], want), float((out[:, 128:256] - want).abs().max())
    assert bool((out[:, :128] == -7.25).all()) and bool((out[:, 256:] == -7.25).all())


def _hand_composition(model, dev, pc, rgb, choose):
    """today's composition of the two engines: torch.gather, FusedPointnet2MSG, FusedHeads"""
    pn2 = mlp.FusedPointnet2MSG(model.pointnet2, dev)
    heads = FusedHeads(model.rgbd_feat, model.SEG_layer, model.KpOF_layer, model.CtrOf_layer, dev)
    with torch.no_grad():
        out_rgb, _ = model.cnn(rgb)
        b, di = out_rgb.shape[:2]
        rgb_emb = torch.gather(out_rgb.view(b, di, -1), 2, choose.repeat(1, di, 1))
        return heads(rgb_emb, pn2(pc))


@pytest.mark.parametrize("b,n", [(2, 4096), (1, 12288)])
def test_fused_network_equals_hand_composition(cuda_dev, b, n):
    model = network_model(n).to(cuda_dev)
    pc, rgb, choose = (t.to(cuda_dev) for t in network_inputs(b, n))
    got = network.FusedPVN3D(model, cuda_dev)(pc, rgb, choose)
    want = _hand_composition(model, cuda_dev, pc, rgb, choose)
    for name, g, w in zip(("kp_of", "seg", "ctr_of"), got, want):
        assert g.shape == w.shape and torch.equal(g, w), name
    assert got[0].shape == (b, 8, n, 3) and got[1].shape == (b, n, 22) and got[2].shape == (b, 1, n, 3)


@pytest.fixture(scope="module")
def network_golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "network_ref.npz")))


@pytest.mark.parametrize("b,n", NETWORK_CASES)
def test_fused_network_matches_reference_forward(cuda_dev, network_golden, b, n):
    model = network_model(n).to(cuda_dev)
    pc, rgb, choose = (t.to(cuda_dev) for t in network_inputs(b, n))
    got = network.FusedPVN3D(model, cuda_dev)(pc, rgb, choose)
    pts = torch.from_numpy(network_points(n)).to(cuda_dev)
    samples = (got[0][:, :, pts], got[1][:, pts], got[2][:, :, pts])
    want = {}
    for name, gt in zip(("kp_of", "seg", "ctr_of"), samples):
        w = torch.from_numpy(network_golden[f"{name}_{b}x{n}"]).to(cuda_dev)
        want[name] = w
        assert gt.shape == w.shape, name
        scale = float(network_golden[f"{name}_{b}x{n}_scale"])
        err = (gt - w).abs()
        print(f"{name} [{b}x{n}]: fused mean {float(err.mean()) / scale:.2e} max {float(err.max()) / scale:.2e}")
        assert float(err.mean()) <= 3e-3 * scale and float(err.max()) <= 3e-2 * scale, name
    top2 = want["seg"].topk(2, dim=-1).values
    clear = (top2[..., 0] - top2[..., 1]) > 1e-2 * float(network_golden[f"seg_{b}x{n}_scale"])
    assert torch.equal(samples[1].argmax(-1)[clear], want["seg"].argmax(-1)[clear])


def test_fused_network_refuses_other_point_counts(cuda_dev):
    model = network_model(4096).to(cuda_dev)
    pc, rgb, choose = (t.to(cuda_dev) for t in network_inputs(1, 2048))
    with pytest.raises(ValueError, match="num_points"):
        network.FusedPVN3D(model, cuda_dev)(pc, rgb, choose)


# ---- compat.patch_pvn3d_forward -------------------------------------------------------------------------------------


@pytest.fixture
def patched_cls():
    cls = type("PatchedStandIn", (testing.StandInPVN3D,), {})
    compat.patch_pvn3d_forward(cls)
    return cls


def _patched_model(cls, n, dev):
    m = cls.__new__(cls)
    m.__dict__.update(network_model(n).__dict__)
    return m.to(dev).eval()


def test_patch_takes_the_fused_path_in_eval_no_grad(cuda_dev, patched_cls):
    b, n = 1, 4096
    m = _patched_model(patched_cls, n, cuda_dev)
    x = [t.to(cuda_dev) for t in network_inputs(b, n)]
    lib = _lib.load()
    eng = network.FusedPVN3D(m, cuda_dev)
    with torch.no_grad():
        want = eng(*x)                                     # warm: every kernel's one-time set-up is done
        torch.cuda.synchronize()
        c0 = lib.pvn3d_launch_count()
        want = eng(*x)
        fused_launches = lib.pvn3d_launch_count() - c0
        m(*x)                                              # builds the cached engine
        c1 = lib.pvn3d_launch_count()
        got = m(*x)
        assert lib.pvn3d_launch_count() - c1 == fused_launches
    assert all(torch.equal(g, w) for g, w in zip(got, want))
    assert compat.fused_engine(m, cuda_dev) is compat.fused_engine(m, cuda_dev)


def test_patch_leaves_training_and_autograd_to_the_original(cuda_dev, patched_cls):
    b, n = 1, 4096
    m = _patched_model(patched_cls, n, cuda_dev)
    x = [t.to(cuda_dev) for t in network_inputs(b, n)]
    orig = patched_cls.forward._pvn3d_b200_orig
    with torch.no_grad():
        m.train()
        got, want = m(*x), orig(m, *x)                     # batch statistics: identical inputs give identical outputs
        assert all(torch.equal(g, w) for g, w in zip(got, want))
        m.eval()
    got = m(*x)                                            # grad enabled
    want = orig(m, *x)
    assert got[0].requires_grad
    assert all(torch.equal(g, w) for g, w in zip(got, want))
    assert "_pvn3d_b200_engines" not in m.__dict__


def test_patch_rebuilds_the_engine_for_new_weights(cuda_dev, patched_cls):
    b, n = 1, 4096
    m = _patched_model(patched_cls, n, cuda_dev)
    x = [t.to(cuda_dev) for t in network_inputs(b, n)]
    with torch.no_grad():
        before = m(*x)
        eng = compat.fused_engine(m, cuda_dev)
        other = testing.StandInPVN3D(n, seed=9)
        m.load_state_dict(other.state_dict())
        after = m(*x)
        assert compat.fused_engine(m, cuda_dev) is not eng
        want = network.FusedPVN3D(other.to(cuda_dev).eval(), cuda_dev)(*x)
    assert all(torch.equal(g, w) for g, w in zip(after, want))
    assert not torch.equal(after[1], before[1])


def test_patch_replica_on_the_source_device_hits_the_cache(cuda_dev, patched_cls):
    b, n = 1, 4096
    m = _patched_model(patched_cls, n, cuda_dev)
    x = [t.to(cuda_dev) for t in network_inputs(b, n)]
    with torch.no_grad():
        want = m(*x)
        eng = compat.fused_engine(m, cuda_dev)
        replica = torch.nn.parallel.replicate(m, [cuda_dev.index or 0])[0]
        got = replica(*x)
        assert compat.fused_engine(replica, cuda_dev) is eng
    assert all(torch.equal(g, w) for g, w in zip(got, want))


def _convert_model(model):
    """the reference's sync_batchnorm.convert_model (demo.py:169) where it is staged, else the same substitution:
    every BatchNorm replaced by an instance of a _BatchNorm subclass sharing its statistics"""
    from helpers import load_reference_python

    if load_reference_python() is not None:
        from lib.utils.sync_batchnorm import convert_model

        return convert_model(model)

    class SyncBN1d(torch.nn.BatchNorm1d):
        pass

    class SyncBN2d(torch.nn.BatchNorm2d):
        pass

    def conv(mod):
        for name, child in mod.named_children():
            for src, dst in ((torch.nn.BatchNorm1d, SyncBN1d), (torch.nn.BatchNorm2d, SyncBN2d)):
                if type(child) is src:
                    new = dst(child.num_features, child.eps, child.momentum, child.affine)
                    new.load_state_dict(child.state_dict())
                    setattr(mod, name, new)
                    break
            else:
                conv(child)
        return mod

    return conv(model)


def test_patch_works_on_a_converted_model(cuda_dev, patched_cls):
    b, n = 1, 4096
    x = [t.to(cuda_dev) for t in network_inputs(b, n)]
    plain = _patched_model(patched_cls, n, cuda_dev)
    with torch.no_grad():
        want = plain(*x)
    m = _convert_model(_patched_model(patched_cls, n, "cpu")).to(cuda_dev).eval()
    bns = [mod for mod in m.modules() if isinstance(mod, torch.nn.modules.batchnorm._BatchNorm)]
    assert bns and all(type(mod).__name__.startswith("Sync") for mod in bns)
    with torch.no_grad():
        got = m(*x)
    assert all(torch.equal(g, w) for g, w in zip(got, want))


def test_patch_refuses_other_point_counts(cuda_dev, patched_cls):
    m = _patched_model(patched_cls, 4096, cuda_dev)
    x = [t.to(cuda_dev) for t in network_inputs(1, 2048)]
    with torch.no_grad(), pytest.raises(ValueError, match="num_points"):
        m(*x)


def test_fused_network_feeds_the_pose_solver(cuda_dev):
    """FusedPVN3D -> seg argmax -> cal_frame_poses on device (demo.py:98-119): finite poses"""
    b, n = 1, 4096
    model = network_model(n).to(cuda_dev)
    pc, rgb, choose = (t.to(cuda_dev) for t in network_inputs(b, n))
    kp_of, seg, ctr_of = network.FusedPVN3D(model, cuda_dev)(pc, rgb, choose)
    mask = eval_utils.seg_argmax(seg)
    s = FramePoseSolver(b, n, 8, 22, fixtures.mesh_kps_table_ycb(), fixtures.radius_thresholds_ycb(), True, device=cuda_dev)
    poses, present, _, _ = s.solve(pc[..., :3].contiguous(), mask, ctr_of[:, 0].contiguous(), kp_of)
    torch.cuda.synchronize()
    assert poses.shape == (b, 22, 3, 4) and bool(torch.isfinite(poses).all())
