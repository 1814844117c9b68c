"""pvn3d_mlp_sa_fact2w (layers 2 and 3 of a factored SA scale with a wide last layer + max-pool, the layer-2
activations kept in shared memory, the weights streamed) against the dense layer on the materialised rows
relu(U[idx] - V): layer 2 with ROUND_OUT, layer 3, then the max over nsample (mlp_compose.sa_fact2).  Same operands,
same MMA N and order per output element: the results must be identical, bit for bit."""
import pytest
import torch

import mlp_compose as compose
from pvn3d_b200 import mlp

from test_mlp_sa_fact2_gpu import _factored_scale

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("b,n,m,ns,c_feat,widths", [
    (2, 1024, 512, 16, 64, (128, 196, 256)),    # SA3 scale 0: layer-2 n_pad 208, layer-3 K 224 (H zero-padded)
    (2, 1024, 512, 32, 64, (128, 196, 256)),    # SA3 scale 1: a centre spans two warps
    (2, 512, 128, 16, 256, (256, 256, 512)),    # SA4 scale 0: four layer-3 blocks
    (2, 512, 128, 32, 256, (256, 384, 512)),    # SA4 scale 1: three layer-2 blocks (uneven warpgroup split)
    (32, 1024, 512, 32, 64, (128, 196, 256)),   # many tiles per persistent CTA: the weight ring and the A tile wrap
    (32, 512, 128, 32, 256, (256, 384, 512)),
    (3, 700, 129, 16, 64, (128, 196, 256)),     # row count not a multiple of 64: ragged last tile
    (3, 700, 129, 32, 256, (256, 384, 512)),
])
@pytest.mark.parametrize("round_out", [False, True])
def test_sa_fact2w_equals_dense_layers_and_max_pool(cuda_dev, b, n, m, ns, c_feat, widths, round_out):
    u, v, idx, l2, l3 = _factored_scale(cuda_dev, b, n, m, ns, c_feat, widths, seed=b + m + ns)
    assert mlp.sa_fact2w_fits(l2, l3, ns)
    want = compose.sa_fact2(u, v, idx, n, l2, l3, round_out=round_out)
    got = mlp.mlp_sa_fact2w(u, v, idx, n, l2, l3, round_out=round_out)
    assert got.shape == want.shape == (b * m, l3.n_pad)
    assert torch.equal(got, want), float((got - want).abs().max())


@pytest.mark.parametrize("ns,c_feat,widths", [(16, 64, (128, 196, 256)), (32, 256, (256, 384, 512))])
def test_sa_fact2w_column_slice_equals_dense_layers(cuda_dev, ns, c_feat, widths):
    b, n, m = 2, 1000, 300
    u, v, idx, l2, l3 = _factored_scale(cuda_dev, b, n, m, ns, c_feat, widths, seed=11 + ns)
    ld, col0 = l3.n_pad + 264, 256
    want = torch.full((b * m, ld), -7.0, device=cuda_dev)
    got = want.clone()
    compose.sa_fact2(u, v, idx, n, l2, l3, round_out=True, out=want, col0=col0)
    mlp.mlp_sa_fact2w(u, v, idx, n, l2, l3, out=got, col0=col0, round_out=True)
    assert torch.equal(got, want)
    assert bool((got[:, :col0] == -7.0).all()) and bool((got[:, col0 + l3.n_pad:] == -7.0).all())


def test_sa_fact2w_rejects_what_it_does_not_cover(cuda_dev):
    u, v, idx, l2, l3 = _factored_scale(cuda_dev, 1, 512, 64, 8, 64, (128, 196, 256), seed=3)
    assert not mlp.sa_fact2w_fits(l2, l3, 8)
    with pytest.raises(mlp._lib.Pvn3dError, match="unsupported"):
        mlp.mlp_sa_fact2w(u, v, idx, 512, l2, l3)
