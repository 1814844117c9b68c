"""The wgmma shared-MLP layer kernel (csrc/mlp_tc.cu) against a float64 torch reference of the same
op on TF32-rounded operands, and the fused hot path A against features recorded from the REFERENCE
Pointnet2MSG.  Tolerances: the kernel itself 2e-5 relative (fp32 accumulation order only); end to end
the TF32 class of the reference's default cuDNN path (written at the assertion)."""
import os

import numpy as np
import pytest
import torch

from pvn3d_b200 import mlp, testing

pytestmark = pytest.mark.gpu


def ref_dense(a, w, b, relu):
    y = a.double() @ w.double().t() + b.double()
    if relu:
        y = y.clamp_min(0)
    return y.float()


@pytest.mark.parametrize("rows,k,n,relu", [
    (128, 32, 16, False), (300, 64, 64, True), (1000, 96, 128, True), (512, 128, 196, True),
    (512, 256, 384, True), (640, 544, 256, True), (2048, 384, 512, True), (1024, 64, 32, True),
    (256, 32, 16, False), (131, 48, 80, True),
    # many tiles per persistent CTA (ring and accumulator tile wrap), odd chunk counts, 2 column blocks
    (64000, 96, 128, True), (70005, 32, 32, True), (40960, 64, 64, True), (9000, 544, 512, True),
    (38400, 160, 272, True),
    # wide layers on 128-column tiles: ragged last tile, 1 / 2 / 4 / 8 column blocks, single-chunk K
    (8192, 96, 128, True), (4144, 64, 128, True), (8000, 224, 256, True), (50016, 224, 256, True),
    (2064, 256, 512, False), (4096, 32, 1024, True), (160, 384, 128, True)])
def test_dense_layer(cuda_dev, rows, k, n, relu):
    g = torch.Generator().manual_seed(rows + k + n)
    a = torch.randn(rows, k, generator=g)
    w = torch.randn(n, k, generator=g) / np.sqrt(k)
    b = torch.randn(n, generator=g)
    layer = mlp.PackedLayer(w.to(cuda_dev), b.to(cuda_dev))
    lda = (k + 15) // 16 * 16
    ad = torch.zeros(rows, lda, device=cuda_dev)
    ad[:, :k] = a.to(cuda_dev)
    out = mlp.mlp_dense(ad, layer, relu=relu).cpu()
    want = ref_dense(mlp.tf32_round(a), mlp.tf32_round(w), b, relu)
    assert out.shape == (rows, layer.n_pad)
    assert (out[:, :n] - want).abs().max() <= 2e-5 * max(1.0, want.abs().max())
    if layer.n_pad > n:
        assert out[:, n:].abs().max() == 0           # pad columns are exact zeros for the next layer


@pytest.mark.parametrize("rows,k,n", [(65536, 96, 128), (32768, 208, 256), (8192, 384, 512)])
def test_layer_into_a_column_slice_of_a_wider_table(cuda_dev, rows, k, n):
    """pre-rounded activations (cp.async producers), the store epilogue writing columns [col0, col0 + n) of a wider
    table, rounded output; the other columns untouched"""
    g = torch.Generator().manual_seed(rows + n)
    a = mlp.tf32_round(torch.randn(rows, k, generator=g)).to(cuda_dev)
    w = torch.randn(n, k, generator=g) / np.sqrt(k)
    b = torch.randn(n, generator=g)
    layer = mlp.PackedLayer(w.to(cuda_dev), b.to(cuda_dev), k)
    table = torch.full((rows, n + 192), 7.0, device=cuda_dev)
    mlp.mlp_dense(a, layer, out=table, col0=64, a_tf32=True, round_out=True)
    want = mlp.tf32_round(ref_dense(a.cpu(), mlp.tf32_round(w), b, True))
    got = table.cpu()
    assert (got[:, 64:64 + n] - want).abs().max() <= 1e-3 * max(1.0, want.abs().max())     # one TF32 ulp of the rounding
    assert (got[:, 64:64 + n] - want).abs().mean() <= 2e-5 * max(1.0, want.abs().max())
    assert torch.equal(got[:, 64:64 + n], mlp.tf32_round(got[:, 64:64 + n]))
    assert (got[:, :64] == 7.0).all() and (got[:, 64 + n:] == 7.0).all()


@pytest.mark.parametrize("rows,k,n1,n2", [(50000, 64, 96, 128), (3000, 256, 384, 512), (20000, 32, 16, 32)])
def test_chained_layers_take_tf32_activations_asynchronously(cuda_dev, rows, k, n1, n2):
    """layer 1 stores TF32-rounded activations (ROUND_OUT), layer 2 copies them with cp.async (A_TF32):
    same numbers as rounding while staging."""
    g = torch.Generator().manual_seed(rows + k)
    a = torch.randn(rows, k, generator=g)
    w1 = torch.randn(n1, k, generator=g) / np.sqrt(k)
    w2 = torch.randn(n2, n1, generator=g) / np.sqrt(n1)
    b1, b2 = torch.randn(n1, generator=g), torch.randn(n2, generator=g)
    l1 = mlp.PackedLayer(w1.to(cuda_dev), b1.to(cuda_dev))
    l2 = mlp.PackedLayer(w2.to(cuda_dev), b2.to(cuda_dev), l1.n_pad)
    ad = torch.zeros(rows, (k + 15) // 16 * 16, device=cuda_dev)
    ad[:, :k] = a.to(cuda_dev)
    h = mlp.mlp_dense(ad, l1, round_out=True)
    assert torch.equal(h, mlp.tf32_round(h))
    h_plain = mlp.mlp_dense(ad, l1)
    assert torch.equal(h, mlp.tf32_round(h_plain))
    out = mlp.mlp_dense(h, l2, a_tf32=True)
    out_sync = mlp.mlp_dense(h_plain, l2)
    assert torch.equal(out, out_sync)
    want = ref_dense(h.cpu()[:, :n1], mlp.tf32_round(w2), b2, True)
    assert (out.cpu()[:, :n2] - want).abs().max() <= 2e-5 * max(1.0, want.abs().max())


def test_fused_pointnet2msg_matches_reference_features(cuda_dev, golden_dir):
    """End to end vs the reference Pointnet2MSG (fp32 on CPU).  TF32 operands (10-bit mantissa) through
    12 shared-MLP layers on raw 0..255 colours: mean error <= 0.3 % and max error <= 5 % of the mean
    feature magnitude -- the same class as the module graph under torch's default TF32 convolutions,
    which is measured alongside."""
    z = np.load(os.path.join(golden_dir, "pn2msg.npz"))
    model = testing.seeded_pointnet2msg(0, 1)
    eng = mlp.FusedPointnet2MSG(model, cuda_dev)
    x = torch.from_numpy(z["cld_rgb_nrm"])[None].to(cuda_dev)
    y = eng(x)
    assert y.shape == (1, 128, x.size(1))
    cols = torch.from_numpy(z["cols"]).long().to(cuda_dev)
    got = y[0][:, cols].cpu().numpy()
    scale = float(z["feat_abs_mean"])
    err = np.abs(got - z["feats"])
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = True
    try:
        with torch.no_grad():
            y_mod = model.to(cuda_dev)(x)[0][:, cols].cpu().numpy()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    err_mod = np.abs(y_mod - z["feats"])
    print(f"fused: mean {err.mean() / scale:.2e} max {err.max() / scale:.2e} | cuDNN-TF32 modules: "
          f"mean {err_mod.mean() / scale:.2e} max {err_mod.max() / scale:.2e}")
    assert err.mean() <= 3e-3 * scale and err.max() <= 5e-2 * scale


def test_fused_engine_is_deterministic(cuda_dev):
    """whole hot path A on the default engine: 200 repetitions of one forward give identical bits (stress for the
    warp-specialised mbarrier pipelines of the per-layer and fused SA kernels)."""
    from pvn3d_b200 import synth

    model = testing.seeded_pointnet2msg(0, 1)
    frames = synth.make_batch("ycb", 2, n_points=12288, config_id=13)
    x = torch.from_numpy(np.stack([f.cld_rgb_nrm for f in frames])).to(cuda_dev)
    eng = mlp.FusedPointnet2MSG(model, cuda_dev)
    y0 = eng(x).clone()
    for i in range(200):
        assert torch.equal(eng(x), y0), f"run {i} differs"


@pytest.mark.parametrize("b,n,m,ns,c_feat,n1", [(2, 1024, 300, 16, 96, 64), (1, 512, 100, 32, 6, 32), (3, 700, 129, 8, 256, 128),
                                                 (2, 2048, 512, 32, 512, 256)])
def test_factored_sa_first_layer_kernels(cuda_dev, b, n, m, ns, c_feat, n1):
    """pvn3d_sa_factor_table + pvn3d_mlp_dense (U) + pvn3d_sa_centre_term (V): U[idx] - V == W1.[f | x - c] + b1 to fp32
    accuracy (the hi/lo coordinate split).  The layers on relu(U[idx] - V) run in the fused SA kernels, which
    test_mlp_fused_f64_gpu.py holds to float64 references."""
    rng = np.random.default_rng(b + n + ns)
    xyz = torch.from_numpy(rng.uniform(-0.5, 1.2, (b, n, 3)).astype(np.float32)).to(cuda_dev)
    sel = torch.from_numpy(np.stack([rng.choice(n, m, replace=False) for _ in range(b)])).to(cuda_dev)
    new_xyz = torch.gather(xyz, 1, sel[..., None].expand(-1, -1, 3)).contiguous()
    idx = torch.from_numpy(rng.integers(0, n, (b, m, ns)).astype(np.int32)).to(cuda_dev)
    feat = torch.from_numpy(rng.normal(size=(b, n, c_feat)).astype(np.float32)).to(cuda_dev)
    g = torch.Generator().manual_seed(n + m)
    w1 = (torch.randn(n1, c_feat + 3, generator=g) / np.sqrt(c_feat + 3)).to(cuda_dev)     # producer order [f | xyz]
    b1 = (torch.randn(n1, generator=g) * 0.1).to(cuda_dev)
    first = mlp.PackedLayer(torch.cat([w1, w1[:, c_feat:]], 1), torch.zeros_like(b1))         # [W_f | W_x | W_x]
    wx = mlp.tf32_round(w1[:, c_feat:].contiguous())
    wxp = torch.zeros((first.n_pad, 3), device=cuda_dev); wxp[:n1] = wx
    b1p = torch.zeros((first.n_pad,), device=cuda_dev); b1p[:n1] = b1
    table = mlp.sa_factor_table(xyz, feat.data_ptr(), c_feat, c_feat, first.k_pad)
    u = mlp.mlp_dense(table, first, relu=False, a_tf32=True)
    v = mlp.sa_centre_term(new_xyz, wxp, b1p)
    bi = torch.arange(b, device=cuda_dev)[:, None, None]
    got1 = (u.view(b, n, -1)[bi, idx.long()] - v.view(b, m, 1, -1))[..., :n1]                  # pre-ReLU first layer
    f64 = mlp.tf32_round(feat).double()[bi, idx.long()]
    dx = xyz.double()[bi, idx.long()] - new_xyz.double()[:, :, None, :]
    want1 = f64 @ mlp.tf32_round(w1[:, :c_feat]).double().t() + dx @ wx.double().t() + b1.double()
    assert float((got1.double() - want1).abs().max()) <= 2e-5 * max(1.0, float(want1.abs().max()))
