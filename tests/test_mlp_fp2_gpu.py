"""pvn3d_mlp_fp2 (both layers of a two-layer FP module in one launch: interpolation fused into the operand producer,
the layer-1 activations kept in shared memory, the weights streamed) against the two launches it replaces:
pvn3d_mlp_fp_first with ROUND_OUT, then pvn3d_mlp_dense.  Same operands, the same MMA N and K order per output element
and the same epilogue arithmetic: the results must be identical, bit for bit."""
import pytest
import torch

from pvn3d_b200 import mlp

pytestmark = pytest.mark.gpu


def _module(dev, b, n, m, c2, c1, n1, n2, seed, lds=None):
    g = torch.Generator().manual_seed(seed)
    lds = c1 if lds is None else lds
    known = torch.randn(b, m, c2, generator=g)
    skip = torch.randn(b * n, max(lds, 1), generator=g)
    nn_idx = torch.randint(0, m, (b, n, 3), generator=g, dtype=torch.int32)
    w = torch.rand(b, n, 3, generator=g) + 0.05
    w = w / w.sum(-1, keepdim=True)
    l1 = mlp.PackedLayer(torch.randn(n1, c2 + c1, generator=g) * (c2 + c1) ** -0.5, torch.randn(n1, generator=g) * 0.1)
    l2 = mlp.PackedLayer(torch.randn(n2, n1, generator=g) * n1 ** -0.5, torch.randn(n2, generator=g) * 0.1, l1.n_pad)
    l1.w, l1.bias, l2.w, l2.bias = (t.to(dev) for t in (l1.w, l1.bias, l2.w, l2.bias))
    return known.to(dev), skip.to(dev), nn_idx.to(dev), w.to(dev), lds, l1, l2


def _two_launches(known, skip, nn_idx, nn_w, lds, c1, l1, l2, round_out=False, reserve=0):
    h = mlp.mlp_fp_first(known, nn_idx, nn_w, skip.data_ptr(), lds, c1, l1, round_out=True, reserve=reserve)
    return mlp.mlp_dense(h, l2, a_tf32=True, round_out=round_out, reserve=reserve)


@pytest.mark.parametrize("b,n,m,c2,c1,n1,n2", [
    (32, 512, 128, 1024, 512, 512, 512),     # FP4 at 32 frames: two passes over K, the rings wrap many times
    (32, 1024, 512, 512, 256, 512, 512),     # FP3
    (32, 2048, 1024, 512, 96, 256, 256),     # FP2: one pass
    (1, 1000, 300, 512, 96, 256, 256),       # rows not a multiple of 64: ragged last tile
    (3, 1000, 257, 1024, 512, 512, 512),
    (3, 700, 129, 80, 52, 256, 384),         # K chunk 2 straddles interpolated / skip columns (generic producer path);
                                             # three layer-2 blocks: the second warpgroup sits the last one out
])
@pytest.mark.parametrize("reserve", [0, 120])
def test_fp2_equals_two_launches(cuda_dev, b, n, m, c2, c1, n1, n2, reserve):
    known, skip, nn_idx, nn_w, lds, l1, l2 = _module(cuda_dev, b, n, m, c2, c1, n1, n2, seed=b + n + c2)
    assert mlp.fp2_fits(l1, l2)
    want = _two_launches(known, skip, nn_idx, nn_w, lds, c1, l1, l2, reserve=reserve)
    got = mlp.mlp_fp2(known, nn_idx, nn_w, skip.data_ptr(), lds, c1, l1, l2, reserve=reserve)
    assert got.shape == want.shape == (b * n, l2.n_pad)
    assert torch.equal(got, want), float((got - want).abs().max())


def test_fp2_unaligned_skip_rows_and_rounded_output(cuda_dev):
    """skip rows 4-byte aligned only (lds odd): every skip chunk takes the generic path; ROUND_OUT on the output"""
    known, skip, nn_idx, nn_w, lds, l1, l2 = _module(cuda_dev, 2, 640, 200, 512, 96, 256, 256, seed=5, lds=97)
    want = _two_launches(known, skip, nn_idx, nn_w, lds, 96, l1, l2, round_out=True)
    got = mlp.mlp_fp2(known, nn_idx, nn_w, skip.data_ptr(), lds, 96, l1, l2, round_out=True)
    assert torch.equal(got, want)


def test_fp2_writes_a_column_slice(cuda_dev):
    b, n, m, c2, c1 = 2, 1000, 300, 512, 256
    known, skip, nn_idx, nn_w, lds, l1, l2 = _module(cuda_dev, b, n, m, c2, c1, 512, 512, seed=17)
    ld, col0 = l2.n_pad + 136, 64
    want = torch.full((b * n, ld), -7.0, device=cuda_dev)
    got = want.clone()
    want[:, col0:col0 + l2.n_pad] = _two_launches(known, skip, nn_idx, nn_w, lds, c1, l1, l2)
    mlp.mlp_fp2(known, nn_idx, nn_w, skip.data_ptr(), lds, c1, l1, l2, out=got, col0=col0)
    assert torch.equal(got, want)


def test_fp2_rejects_what_it_does_not_cover(cuda_dev):
    known, skip, nn_idx, nn_w, lds, l1, l2 = _module(cuda_dev, 1, 256, 64, 256, 6, 128, 128, seed=3)
    assert not mlp.fp2_fits(l1, l2)
    with pytest.raises(mlp._lib.Pvn3dError, match="unsupported"):
        mlp.mlp_fp2(known, nn_idx, nn_w, skip.data_ptr(), lds, 6, l1, l2)
