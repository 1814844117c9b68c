"""pvn3d_mlp_sa_fact2 (layers 2 and 3 of a factored SA scale + max-pool, the layer-2 activations kept in shared
memory) against the dense layer on the materialised rows relu(U[idx] - V): layer 2 with ROUND_OUT, layer 3, then the
max over nsample (mlp_compose.sa_fact2).  Same operands, same MMA order per output element: the results must be
identical, bit for bit."""
import numpy as np
import pytest
import torch

import mlp_compose as compose
from pvn3d_b200 import mlp

pytestmark = pytest.mark.gpu


def _factored_scale(dev, b, n, m, ns, c_feat, widths, seed):
    rng = np.random.default_rng(seed)
    xyz = torch.from_numpy(rng.uniform(-0.5, 1.2, (b, n, 3)).astype(np.float32)).to(dev)
    sel = torch.from_numpy(np.stack([rng.choice(n, m, replace=False) for _ in range(b)])).to(dev)
    new_xyz = torch.gather(xyz, 1, sel[..., None].expand(-1, -1, 3)).contiguous()
    idx = torch.from_numpy(rng.integers(0, n, (b, m, ns)).astype(np.int32)).to(dev)
    feat = torch.from_numpy(rng.normal(size=(b, n, c_feat)).astype(np.float32)).to(dev)
    g = torch.Generator().manual_seed(seed)
    n1, n2, n3 = widths
    w1 = (torch.randn(n1, c_feat + 3, generator=g) / np.sqrt(c_feat + 3)).to(dev)
    b1 = (torch.randn(n1, generator=g) * 0.1).to(dev)
    first = mlp.PackedLayer(torch.cat([w1, w1[:, c_feat:]], 1), torch.zeros_like(b1))
    wx = torch.zeros((first.n_pad, 3), device=dev)
    wx[:n1] = mlp.tf32_round(w1[:, c_feat:].contiguous())
    b1p = torch.zeros((first.n_pad,), device=dev)
    b1p[:n1] = b1
    table = mlp.sa_factor_table(xyz, feat.data_ptr(), c_feat, c_feat, first.k_pad)
    u = mlp.mlp_dense(table, first, relu=False, a_tf32=True)
    v = mlp.sa_centre_term(new_xyz, wx, b1p)
    l2 = mlp.PackedLayer((torch.randn(n2, n1, generator=g) / np.sqrt(n1)).to(dev), (torch.randn(n2, generator=g) * 0.1).to(dev),
                         first.n_pad)
    l3 = mlp.PackedLayer((torch.randn(n3, n2, generator=g) / np.sqrt(n2)).to(dev), (torch.randn(n3, generator=g) * 0.1).to(dev),
                         l2.n_pad)
    return u, v, idx, l2, l3


@pytest.mark.parametrize("b,n,m,ns,c_feat,widths", [
    (2, 12288, 2048, 16, 6, (16, 16, 32)),     # SA1 scale 0: one K chunk per layer, layer-2 MMA narrower than layer 3's K
    (2, 12288, 2048, 32, 6, (32, 32, 64)),     # SA1 scale 1: a centre spans two warps
    (2, 2048, 1024, 16, 96, (64, 64, 128)),    # SA2 scale 0: two K chunks per layer
    (2, 2048, 1024, 32, 96, (64, 96, 128)),    # SA2 scale 1: n_pad 96 (wgmma N 128, layer-3 K 96)
    (3, 700, 129, 16, 96, (64, 64, 128)),      # row count not a multiple of 128: ragged last tile
    (3, 700, 129, 32, 6, (32, 32, 64)),
    (32, 2048, 1024, 32, 6, (32, 32, 64)),     # many tiles per persistent CTA: the operand ring wraps
    (2, 1024, 300, 16, 6, (256, 64, 128)),     # 8 layer-2 K chunks per tile, more than the ring's 5 stages
    (2, 1024, 300, 32, 6, (256, 32, 64)),
])
@pytest.mark.parametrize("round_out", [False, True])
def test_sa_fact2_equals_dense_layers_and_max_pool(cuda_dev, b, n, m, ns, c_feat, widths, round_out):
    u, v, idx, l2, l3 = _factored_scale(cuda_dev, b, n, m, ns, c_feat, widths, seed=b + m + ns)
    want = compose.sa_fact2(u, v, idx, n, l2, l3, round_out=round_out)
    got = mlp.mlp_sa_fact2(u, v, idx, n, l2, l3, round_out=round_out)
    assert got.shape == want.shape == (b * m, l3.n_pad)
    assert torch.equal(got, want), float((got - want).abs().max())


@pytest.mark.parametrize("ns,c_feat,widths", [(16, 96, (64, 64, 128)), (32, 6, (32, 32, 64))])
def test_sa_fact2_column_slice_equals_dense_layers(cuda_dev, ns, c_feat, widths):
    b, n, m = 2, 1000, 300
    u, v, idx, l2, l3 = _factored_scale(cuda_dev, b, n, m, ns, c_feat, widths, seed=7 + ns)
    ld, col0 = l3.n_pad + 72, 40
    want = torch.full((b * m, ld), -7.0, device=cuda_dev)
    got = want.clone()
    compose.sa_fact2(u, v, idx, n, l2, l3, round_out=True, out=want, col0=col0)
    mlp.mlp_sa_fact2(u, v, idx, n, l2, l3, out=got, col0=col0, round_out=True)
    assert torch.equal(got, want)
    assert bool((got[:, :col0] == -7.0).all()) and bool((got[:, col0 + l3.n_pad:] == -7.0).all())


def test_sa_fact2_rejects_what_it_does_not_cover(cuda_dev):
    u, v, idx, l2, l3 = _factored_scale(cuda_dev, 1, 512, 64, 8, 6, (16, 16, 32), seed=3)
    assert not mlp.sa_fact2_fits(l2, l3, 8)
    with pytest.raises(mlp._lib.Pvn3dError, match="unsupported"):
        mlp.mlp_sa_fact2(u, v, idx, 512, l2, l3)
