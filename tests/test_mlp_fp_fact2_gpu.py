"""pvn3d_mlp_fp_fact2 (the skip term S = W1s . table + b1 and the second layer of a factored FP module in one launch, S
kept on chip, the output stored channel-major) against the dense layer without ReLU on the SA1 factor table for S, then
the dense layer on the materialised rows relu(three_interpolate(P) + S), transposed per frame (mlp_compose.fp_fact2).
Same operands, the same MMA shape and K order per output element and the same epilogue arithmetic: the results must be
identical, bit for bit."""
import pytest
import torch

import mlp_compose as compose
from pvn3d_b200 import mlp

pytestmark = pytest.mark.gpu


def _module(dev, b, n, m, seed, c_feat=6):
    g = torch.Generator().manual_seed(seed)
    xyz = (torch.rand(b, n, 3, generator=g) * 2 - 1).to(dev)
    feat = torch.randn(b * n, c_feat, generator=g).to(dev)
    p = (torch.randn(b * m, 128, generator=g) * 0.5).to(dev)
    nn_idx = torch.randint(0, m, (b, n, 3), generator=g, dtype=torch.int32).to(dev)
    w = torch.rand(b, n, 3, generator=g) + 0.05
    nn_w = (w / w.sum(-1, keepdim=True)).to(dev)
    # the skip layer reads [f | hi x | lo x]: the coordinate columns meet the same weights twice, as the engine packs it
    ws = torch.randn(128, c_feat + 3, generator=g) * (c_feat + 3) ** -0.5
    ls = mlp.PackedLayer(torch.cat([ws, ws[:, c_feat:]], dim=1), torch.randn(128, generator=g) * 0.1)
    l2 = mlp.PackedLayer(torch.randn(128, 128, generator=g) * 128 ** -0.5, torch.randn(128, generator=g) * 0.1, ls.n_pad)
    ls.w, ls.bias, l2.w, l2.bias = (t.to(dev) for t in (ls.w, ls.bias, l2.w, l2.bias))
    table = mlp.sa_factor_table(xyz, feat.data_ptr(), c_feat, c_feat, ls.k_pad)
    return p, table, nn_idx, nn_w, ls, l2


@pytest.mark.parametrize("b,n,m", [
    (32, 12288, 2048),   # the bench shape
    (3, 1000, 333),      # frames end inside tiles
    (1, 96, 40),         # one and a half tiles
])
@pytest.mark.parametrize("reserve", [0, 120])
def test_fp_fact2_equals_transposed_dense_layers(cuda_dev, b, n, m, reserve):
    p, table, nn_idx, nn_w, ls, l2 = _module(cuda_dev, b, n, m, seed=b + n + m)
    assert mlp.fp_fact2_fits(ls, l2)
    assert bool((table[:, 6:12] != 0).any())          # the hi / lo coordinate columns take part
    want = compose.fp_fact2(p, table, nn_idx, nn_w, m, ls, l2, reserve=reserve)
    got = mlp.mlp_fp_fact2(p, table, nn_idx, nn_w, m, ls, l2, reserve=reserve)
    assert got.shape == want.shape == (b, 128, n)
    assert torch.equal(got, want), float((got - want).abs().max())


def test_fp_fact2_engine_output_equals_dense_layers(cuda_dev):
    """FusedPointnet2MSG.features: FP1 through the fused launch gives what P -> S -> the dense layer on
    relu(three_interpolate(P) + S) gives"""
    from pvn3d_b200 import synth, testing

    host = synth.stack(synth.make_batch("linemod", 2, n_points=3000, config_id=2, lm_obj_id=1))
    cloud = torch.from_numpy(host["cld_rgb_nrm"]).to(cuda_dev).contiguous()
    eng = mlp.FusedPointnet2MSG(testing.seeded_pointnet2msg(0, 1), cuda_dev)
    plan = eng.geometry(cloud)
    got = eng.features(cloud, plan)
    lk, ls, l2 = eng.fp1
    calls = {}
    orig = mlp.mlp_fp_fact2

    def spy(p, table, nn_idx, nn_w, m_known, layer_s, layer2, reserve=0):
        calls.update(p=p, table=table, nn_idx=nn_idx, nn_w=nn_w, m=m_known)
        return orig(p, table, nn_idx, nn_w, m_known, layer_s, layer2, reserve=reserve)

    mlp.mlp_fp_fact2 = spy
    try:
        again = eng.features(cloud, plan)
    finally:
        mlp.mlp_fp_fact2 = orig
    assert torch.equal(got, again)
    want = compose.fp_fact2(calls["p"], calls["table"], calls["nn_idx"], calls["nn_w"], calls["m"], ls, l2)
    assert torch.equal(got, want)
