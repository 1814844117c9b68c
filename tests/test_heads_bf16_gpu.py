"""The heads in bf16 (FusedHeads(precision="bf16"), FusedPVN3D(precision="bf16"), the PVN3D.forward patch under bf16
autocast) on the device:

  * every bf16 launch against a torch emulation: operands rounded to bf16, fp64 accumulation, bias, ReLU, the stored
    bf16 value rounded once -- stored bf16 values within one bf16 ulp of the exact value plus the fp32 accumulation
    allowance (1e-5 of |A|.|W|^T + |bias|, which only matters where the sum cancels to near zero), >= 99.9 % identical
    to the emulation; f32 outputs and the 32-row sums within that same 1e-5 of the scale;
  * the bf16 producers of the table (the gather, FP1's rows) bit for bit, other columns untouched;
  * the whole heads against the fp32 module graph (TF32 off): no worse than 1.5x the error of the same modules under
    torch.autocast(bfloat16), mean and 99.9th percentile, seg arg-max agreeing where the fp32 margin is clear;
  * FusedPVN3D(precision="bf16") against the hand composition, bit for bit, and into the pose solver;
  * the patch: bf16 autocast -> the bf16 engine, no autocast and fp16 autocast -> the TF32 engine, one cached engine
    per precision.
"""
import pytest
import torch

from pvn3d_b200 import compat, eval_utils, fixtures, heads, mlp, network, testing
from pvn3d_b200._lib import call, ptr
from pvn3d_b200.eval_utils import FramePoseSolver

from helpers import HEADS_CASES, heads_inputs, heads_modules
from network_cases import network_inputs, network_model

pytestmark = pytest.mark.gpu

RELU, OUT_BF16 = 1, 8


@pytest.fixture(autouse=True)
def _fp32_reference():
    """the module-graph references below run in fp32"""
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _bits(x):
    return x.contiguous().view(torch.int16).to(torch.int32)


def _emulate(a_bf16, a_cols, layer, bias, relu):
    """fp64 act(A[:, :a_cols] . W^T + bias) of bf16 operands -> [rows, n_pad] f64"""
    a = a_bf16[:, :a_cols].double()
    acc = a @ layer.w[:, :a_cols].double().t() + bias.double()
    return acc.clamp_min(0) if relu else acc


def _scale(a_bf16, a_cols, layer, bias):
    """|A| . |W|^T + |bias|: the magnitude an fp32 accumulation error is relative to"""
    return a_bf16[:, :a_cols].double().abs() @ layer.w[:, :a_cols].double().abs().t() + bias.double().abs()


def _operands(dev, rows, k, n, a_cols, lda, seed):
    g = torch.Generator().manual_seed(seed)
    layer = mlp.PackedLayer(torch.randn(n, k, generator=g) * k ** -0.5, torch.randn(n, generator=g) * 0.1, precision="bf16")
    layer.w, layer.bias = layer.w.to(dev), layer.bias.to(dev)
    a = torch.full((rows, lda), float("nan"), dtype=torch.bfloat16)    # columns >= a_cols must read as zero
    a[:, :a_cols] = torch.randn(rows, a_cols, generator=g).abs().to(torch.bfloat16)
    return a.to(dev), layer


def _check_bf16_store(got, want, scale):
    """stored bf16 within one bf16 ulp (of the emulation rounded once) of the exact value, plus the fp32 accumulation
    allowance; >= 99.9 % bit-identical to the emulation rounded once"""
    want16 = want.to(torch.bfloat16)
    _, e = torch.frexp(want16.double())
    ulp = torch.where(want16 == 0, torch.zeros_like(want), torch.ldexp(torch.ones_like(want), e - 8))
    err = (got.double() - want).abs()
    bad = err > ulp + 1e-5 * scale
    assert not bool(bad.any()), (int(bad.sum()), float(err[bad].max()))
    same = float((_bits(got) == _bits(want16)).double().mean())
    assert same >= 0.999, same


# (rows, k, n, a_cols, lda): a ragged last row tile, a ragged last 128-column block (n 144), the narrow head outputs
DENSE_CASES = [(1000, 256, 144, 200, 264), (4096, 768, 1024, 768, 1280), (2000, 128, 22, 128, 128),
               (777, 128, 3, 128, 136), (1280, 512, 64, 504, 512)]


@pytest.mark.parametrize("rows,k,n,a_cols,lda", DENSE_CASES)
def test_dense_bf16_store_matches_emulation(cuda_dev, rows, k, n, a_cols, lda):
    a, layer = _operands(cuda_dev, rows, k, n, a_cols, lda, seed=rows + n)
    want = _emulate(a, a_cols, layer, layer.bias, relu=True)
    col0, ldo = 8, layer.n_pad + 16
    out = torch.full((rows, ldo), -7.25, dtype=torch.bfloat16, device=cuda_dev)
    call("pvn3d_mlp_dense_bf16", cuda_dev, ptr(a), lda, a_cols, rows, ptr(layer.w), ptr(layer.bias), layer.k_pad,
         layer.n_pad, RELU | OUT_BF16, ptr(out), ldo, col0)
    _check_bf16_store(out[:, col0:col0 + layer.n_pad], want, _scale(a, a_cols, layer, layer.bias))
    assert bool((out[:, :col0] == -7.25).all()) and bool((out[:, col0 + layer.n_pad:] == -7.25).all())
    # f32 rows, no ReLU (the last layer of a head)
    want = _emulate(a, a_cols, layer, layer.bias, relu=False)
    out32 = torch.empty((rows, layer.n_pad), dtype=torch.float32, device=cuda_dev)
    call("pvn3d_mlp_dense_bf16", cuda_dev, ptr(a), lda, a_cols, rows, ptr(layer.w), ptr(layer.bias), layer.k_pad,
         layer.n_pad, 0, ptr(out32), layer.n_pad, 0)
    err = (out32.double() - want).abs()
    assert bool((err <= 1e-5 * _scale(a, a_cols, layer, layer.bias)).all()), float(err.max())


@pytest.mark.parametrize("frames,n", [(2, 2048), (3, 1280)])
def test_dense_bf16_frame_bias_matches_emulation(cuda_dev, frames, n):
    rows, k, nc = frames * n, 768, 1024
    a, layer = _operands(cuda_dev, rows, k, nc, k, 1280, seed=n)
    fb = torch.randn(frames, layer.n_pad, generator=torch.Generator().manual_seed(7)).to(cuda_dev)
    want = torch.cat([_emulate(a[f * n:(f + 1) * n], k, layer, fb[f], relu=True) for f in range(frames)])
    scale = torch.cat([_scale(a[f * n:(f + 1) * n], k, layer, fb[f]) for f in range(frames)])
    out = torch.empty((rows, layer.n_pad), dtype=torch.bfloat16, device=cuda_dev)
    call("pvn3d_mlp_dense_frame_bias_bf16", cuda_dev, ptr(a), 1280, k, rows, n, ptr(layer.w), ptr(fb), layer.k_pad,
         layer.n_pad, RELU | OUT_BF16, ptr(out), layer.n_pad, 0)
    _check_bf16_store(out, want, scale)


@pytest.mark.parametrize("rows", [4096, 1000])
def test_dense_bf16_sum32_matches_emulation(cuda_dev, rows):
    a, layer = _operands(cuda_dev, rows, 512, 1024, 512, 1280, seed=rows)
    want = _emulate(a, 512, layer, layer.bias, relu=True)
    scale = _scale(a, 512, layer, layer.bias)
    groups = (rows + 31) // 32
    pad = groups * 32 - rows
    want_s = torch.nn.functional.pad(want, (0, 0, 0, pad)).view(groups, 32, -1).sum(1)
    scale_s = torch.nn.functional.pad(scale, (0, 0, 0, pad)).view(groups, 32, -1).sum(1)
    part = torch.empty((groups, layer.n_pad), dtype=torch.float32, device=cuda_dev)
    call("pvn3d_mlp_dense_sum32_bf16", cuda_dev, ptr(a), 1280, 512, rows, ptr(layer.w), ptr(layer.bias), layer.k_pad,
         layer.n_pad, RELU, ptr(part), layer.n_pad, 0)
    err = (part.double() - want_s).abs()
    assert bool((err <= 1e-5 * scale_s).all()), float((err / scale_s).max())
    again = torch.empty_like(part)
    call("pvn3d_mlp_dense_sum32_bf16", cuda_dev, ptr(a), 1280, 512, rows, ptr(layer.w), ptr(layer.bias), layer.k_pad,
         layer.n_pad, RELU, ptr(again), layer.n_pad, 0)
    assert torch.equal(part, again)                                   # fixed summation order


# ---- the bf16 producers of the table ---------------------------------------------------------------------------------


def _gather_ref(emb, choose):
    b, c = emb.shape[:2]
    g = torch.gather(emb.reshape(b, c, -1), 2, choose.repeat(1, c, 1))
    return g.transpose(1, 2).reshape(-1, c).to(torch.bfloat16)


@pytest.mark.parametrize("src", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("b,c,hw,n", [(2, 128, 120 * 160, 4096), (3, 32, 500, 1000)])
def test_gather_pixel_rows_bf16_bit_exact(cuda_dev, src, b, c, hw, n):
    emb = torch.randn(b, c, hw, generator=torch.Generator().manual_seed(c + n)).to(cuda_dev, src)
    choose = testing.sample_choose(b, n, hw, seed=n)
    choose[0, 0, :3] = torch.tensor([0, hw - 1, hw - 1])
    choose = choose.to(cuda_dev)
    col0, ldo = 128, 1280
    out = torch.full((b * n, ldo), -7.25, dtype=torch.bfloat16, device=cuda_dev)
    network.gather_pixel_rows(emb, choose, out, col0=col0)
    assert torch.equal(_bits(out[:, col0:col0 + c]), _bits(_gather_ref(emb, choose)))
    assert bool((out[:, :col0] == -7.25).all()) and bool((out[:, col0 + c:] == -7.25).all())


def test_gather_bf16_out_of_range_index_gives_a_nan_row(cuda_dev):
    b, c, hw, n = 2, 128, 4000, 1000
    emb = torch.randn(b, c, hw, generator=torch.Generator().manual_seed(1)).to(cuda_dev)
    choose = testing.sample_choose(b, n, hw, seed=3)
    choose[1, 0, 999] = hw
    out = torch.zeros((b * n, 256), dtype=torch.bfloat16, device=cuda_dev)
    network.gather_pixel_rows(emb, choose.to(cuda_dev), out, col0=0)
    assert bool(torch.isnan(out[2 * n - 1, :c]).all()) and not bool(torch.isnan(out[: 2 * n - 1]).any())


@pytest.mark.parametrize("b,n,m", [(2, 12288, 2048), (3, 1000, 333)])
def test_fp1_rows_bf16_bit_exact(cuda_dev, b, n, m):
    from test_network_gpu import _fp1_module

    p, table, nn_idx, nn_w, ls, l2 = _fp1_module(cuda_dev, b, n, m, seed=n)
    cn = mlp.mlp_fp_fact2(p, table, nn_idx, nn_w, m, ls, l2)                     # [b, 128, n] f32 (unrounded)
    want = cn.transpose(1, 2).reshape(b * n, 128).to(torch.bfloat16)
    out = torch.full((b * n, 1280), -7.25, dtype=torch.bfloat16, device=cuda_dev)
    mlp.mlp_fp_fact2_rows(p, table, nn_idx, nn_w, m, ls, l2, out, 128)
    assert torch.equal(_bits(out[:, 128:256]), _bits(want))
    assert bool((out[:, :128] == -7.25).all()) and bool((out[:, 256:] == -7.25).all())


# ---- the whole heads -----------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def ref_modules(cuda_dev):
    return [m.to(cuda_dev).eval() for m in heads_modules()]


def _module_graph(mods, rgb_emb, cld_emb):
    """DenseFusion + heads as PVN3D.forward composes them (pvn3d.py:157-182, 297-306; testing.StandInPVN3D)"""
    f = torch.nn.functional
    d, seg_l, kp_l, ctr_l = mods
    bs, _, n = rgb_emb.shape
    feat_1 = torch.cat((rgb_emb, cld_emb), dim=1)
    feat_2 = torch.cat((f.relu(d.conv2_rgb(rgb_emb)), f.relu(d.conv2_cld(cld_emb))), dim=1)
    ap_x = f.relu(d.conv4(f.relu(d.conv3(feat_1)))).mean(2, keepdim=True).repeat(1, 1, n)
    feat = torch.cat([feat_1, feat_2, ap_x], 1)
    seg = seg_l(feat).transpose(1, 2).contiguous()
    kp = kp_l(feat).view(bs, 8, 3, n).permute(0, 1, 3, 2).contiguous()
    ctr = ctr_l(feat).view(bs, 1, 3, n).permute(0, 1, 3, 2).contiguous()
    return kp, seg, ctr


def _err_stats(got, want, scale):
    e = (got.double() - want.double()).abs().flatten() / scale
    return float(e.mean()), float(torch.quantile(e[: 1 << 24], 0.999))


@pytest.mark.parametrize("b,n", HEADS_CASES)
def test_bf16_heads_no_worse_than_autocast(cuda_dev, ref_modules, b, n):
    rgb_emb, cld_emb = (t.to(cuda_dev) for t in heads_inputs(b, n))
    with torch.no_grad():
        want = _module_graph(ref_modules, rgb_emb, cld_emb)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            auto = _module_graph(ref_modules, rgb_emb, cld_emb)
    eng = heads.FusedHeads(*ref_modules, device=cuda_dev, precision="bf16")
    got = eng(rgb_emb, cld_emb)
    for name, g, a, w in zip(("kp_of", "seg", "ctr_of"), got, auto, want):
        assert g.dtype == torch.float32 and g.shape == w.shape and g.is_contiguous(), name
        scale = float(w.abs().mean())
        g_mean, g_p999 = _err_stats(g, w, scale)
        a_mean, a_p999 = _err_stats(a, w, scale)
        print(f"{name} [{b}x{n}]: bf16 engine mean {g_mean:.2e} p99.9 {g_p999:.2e} | autocast mean {a_mean:.2e} "
              f"p99.9 {a_p999:.2e}")
        assert g_mean <= 1.5 * a_mean and g_p999 <= 1.5 * a_p999, name
    seg_w, seg_g = want[1], got[1]
    top2 = seg_w.topk(2, dim=-1).values
    clear = (top2[..., 0] - top2[..., 1]) > 2e-2 * float(seg_w.abs().mean())
    assert torch.equal(seg_g.argmax(-1)[clear], seg_w.argmax(-1)[clear])


def test_bf16_heads_take_bf16_inputs(cuda_dev, ref_modules):
    """bf16 embeddings give the same table, so the same outputs, as their f32 values"""
    rgb_emb, cld_emb = (t.to(cuda_dev).to(torch.bfloat16) for t in heads_inputs(1, 2048))
    eng = heads.FusedHeads(*ref_modules, device=cuda_dev, precision="bf16")
    got, want = eng(rgb_emb, cld_emb), eng(rgb_emb.float(), cld_emb.float())
    assert all(torch.equal(g, w) for g, w in zip(got, want))


# ---- FusedPVN3D and the patch ----------------------------------------------------------------------------------------


@pytest.mark.parametrize("b,n", [(2, 4096), (1, 12288)])
def test_bf16_network_equals_hand_composition(cuda_dev, b, n):
    model = network_model(n).to(cuda_dev)
    pc, rgb, choose = (t.to(cuda_dev) for t in network_inputs(b, n))
    got = network.FusedPVN3D(model, cuda_dev, precision="bf16")(pc, rgb, choose)
    pn2 = mlp.FusedPointnet2MSG(model.pointnet2, cuda_dev)
    hd = heads.FusedHeads(model.rgbd_feat, model.SEG_layer, model.KpOF_layer, model.CtrOf_layer, cuda_dev, "bf16")
    with torch.no_grad():
        out_rgb, _ = model.cnn(rgb)
        rgb_emb = torch.gather(out_rgb.view(b, 128, -1), 2, choose.repeat(1, 128, 1))
        want = hd(rgb_emb, pn2(pc))
    for name, g, w in zip(("kp_of", "seg", "ctr_of"), got, want):
        assert g.dtype == torch.float32 and g.shape == w.shape and torch.equal(g, w), name


def test_bf16_network_feeds_the_pose_solver(cuda_dev):
    b, n = 1, 4096
    model = network_model(n).to(cuda_dev)
    pc, rgb, choose = (t.to(cuda_dev) for t in network_inputs(b, n))
    kp_of, seg, ctr_of = network.FusedPVN3D(model, cuda_dev, precision="bf16")(pc, rgb, choose)
    mask = eval_utils.seg_argmax(seg)
    s = FramePoseSolver(b, n, 8, 22, fixtures.mesh_kps_table_ycb(), fixtures.radius_thresholds_ycb(), True, device=cuda_dev)
    poses, present, _, _ = s.solve(pc[..., :3].contiguous(), mask, ctr_of[:, 0].contiguous(), kp_of)
    torch.cuda.synchronize()
    assert poses.shape == (b, 22, 3, 4) and bool(torch.isfinite(poses).all())


def test_patch_routes_autocast_bf16_to_the_bf16_engine(cuda_dev):
    cls = type("PatchedStandInBf16", (testing.StandInPVN3D,), {})
    compat.patch_pvn3d_forward(cls)
    b, n = 1, 4096
    m = cls.__new__(cls)
    m.__dict__.update(network_model(n).__dict__)
    m = m.to(cuda_dev).eval()
    x = [t.to(cuda_dev) for t in network_inputs(b, n)]
    eng_tf32 = network.FusedPVN3D(m, cuda_dev)
    eng_bf16 = network.FusedPVN3D(m, cuda_dev, precision="bf16")
    with torch.no_grad():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            got, want = m(*x), eng_bf16(*x)               # the CNN runs under autocast in both: a bf16 embedding
        assert all(g.dtype == torch.float32 and torch.equal(g, w) for g, w in zip(got, want))
        got, want = m(*x), eng_tf32(*x)
        assert all(torch.equal(g, w) for g, w in zip(got, want))
        with torch.autocast("cuda", dtype=torch.float16):
            got, want = m(*x), eng_tf32(*x)
        assert all(torch.equal(g, w) for g, w in zip(got, want))
    engines = m.__dict__["_pvn3d_b200_engines"]
    assert set(engines) == {(x[0].device, "tf32"), (x[0].device, "bf16")}
    assert compat.fused_engine(m, x[0].device, "bf16").precision == "bf16"
    assert compat.fused_engine(m, x[0].device).precision == "tf32"
