"""The fused shared-MLP kernels the engine runs, each against a float64 reference of its own operation with an
element-wise bound (tests/f64_bounds.py) -- not only against the two-launch forms that share their producer code:

  * pvn3d_mlp_sa_fact2 (SA1 / SA2): all 16 (layer-2, layer-3) wgmma N instantiations, the production shapes at 32
    frames, a ragged last tile, ROUND_OUT both ways, reserved SMs, a column slice;
  * pvn3d_mlp_sa_fact2w (SA3 / SA4): the production shapes, ragged layer-3 blocks (n3 144, 400), layer-2 widths that
    are not a multiple of 128 (144, 208), a column slice;
  * pvn3d_mlp_fp2 (FP2-FP4): the production shapes, a K chunk across the interpolated / skip boundary, unaligned skip
    rows, layer-2 widths 128 / 384, a column slice;
  * pvn3d_mlp_fp_fact2 and _rows (FP1): the production shape, point counts not a multiple of 8, tiles that span frames.

Every kernel's check is also shown to fail on references that are wrong in the ways a kernel could be."""
import itertools

import pytest
import torch

import f64_bounds as fb
from pvn3d_b200 import mlp

from test_mlp_fp2_gpu import _module as _fp_module
from test_mlp_sa_fact2_gpu import _factored_scale
from test_network_gpu import _fp1_module

pytestmark = pytest.mark.gpu


def _n_pad(n):
    return (n + 15) // 16 * 16


def _mma_n(n_pad):
    """the wgmma N a layer of n_pad columns runs at (mma_n in csrc/mlp_tc.cu)"""
    return 16 if n_pad <= 16 else 32 if n_pad <= 32 else 64 if n_pad <= 64 else 128


# ---- SA: layers 2 and 3 + max-pool ----------------------------------------------------------------------------------


def _sa_rows(idx, n, m):
    """U row and V row of every grouped row (centre-major)"""
    b, _, ns = idx.shape
    frame = torch.arange(b, device=idx.device)[:, None, None]
    rows_u = (frame * n + idx.long()).reshape(-1)
    rows_v = torch.arange(b * m, device=idx.device).repeat_interleave(ns)
    return rows_u, rows_v


def _sa_ref(u, v, idx, n, l2, l3, round_out):
    rows_u, rows_v = _sa_rows(idx, n, idx.size(1))
    return fb.sa_scale(u, v, rows_u, rows_v, l2.w, l2.bias, l3.w, l3.bias, idx.size(2), round_out)


def _sa_check(dev, fused, fits, b, n, m, ns, c_feat, widths, round_out, reserve=0, seed=0, slice_=False):
    u, v, idx, l2, l3 = _factored_scale(dev, b, n, m, ns, c_feat, widths, seed=seed)
    assert fits(l2, l3, ns), (widths, ns)
    ref, bound = _sa_ref(u, v, idx, n, l2, l3, round_out)
    name = f"{fused.__name__} b{b} m{m} ns{ns} {widths} round_out={round_out}"
    if not slice_:
        got = fused(u, v, idx, n, l2, l3, round_out=round_out, reserve=reserve)
        fb.check(got, ref, bound, name)
        return
    col0, ld = 40, l3.n_pad + 72
    out = torch.full((b * m, ld), -7.0, device=dev)
    fused(u, v, idx, n, l2, l3, out=out, col0=col0, round_out=round_out, reserve=reserve)
    fb.check(out[:, col0:col0 + l3.n_pad], ref, bound, name + " slice")
    assert bool((out[:, :col0] == -7.0).all()) and bool((out[:, col0 + l3.n_pad:] == -7.0).all())


# every (mma_n(l2.n_pad), mma_n(l3.n_pad)) instantiation of mlp_sa_fact2_kernel, the layer-2 K (n1) from 16 to 256,
# nsample 16 and 32, ROUND_OUT and the reserved SMs alternating
_SA2_K = (16, 32, 64, 96, 128, 256, 48, 160)
SA2_PAIRS = [((_SA2_K[i % len(_SA2_K)], n2, n3), (16, 32)[i % 2], bool(i % 3 == 0), (0, 120)[(i // 2) % 2])
             for i, (n2, n3) in enumerate(itertools.product((16, 32, 48, 96), (16, 32, 64, 112)))]
assert {(_mma_n(_n_pad(w[1])), _mma_n(_n_pad(w[2]))) for w, _, _, _ in SA2_PAIRS} == set(
    itertools.product((16, 32, 64, 128), repeat=2)), "the cases must reach every mlp_sa_fact2_kernel<N2, N3>"


@pytest.mark.parametrize("widths,ns,round_out,reserve", SA2_PAIRS)
def test_sa_fact2_instantiations_within_f64_bound(cuda_dev, widths, ns, round_out, reserve):
    _sa_check(cuda_dev, mlp.mlp_sa_fact2, mlp.sa_fact2_fits, 2, 1024, 256, ns, 6 if widths[0] < 64 else 96, widths,
              round_out, reserve, seed=sum(widths) + ns)


@pytest.mark.parametrize("b,n,m,ns,c_feat,widths", [
    (32, 12288, 2048, 16, 6, (16, 16, 32)),    # SA1 at 32 frames: the operand ring wraps
    (32, 12288, 2048, 32, 6, (32, 32, 64)),
    (32, 2048, 1024, 16, 96, (64, 64, 128)),   # SA2
    (32, 2048, 1024, 32, 96, (64, 96, 128)),
    (3, 700, 129, 16, 96, (64, 64, 128)),      # a ragged last tile
    (3, 700, 129, 32, 6, (32, 32, 64)),
])
@pytest.mark.parametrize("round_out", [False, True])
def test_sa_fact2_production_shapes_within_f64_bound(cuda_dev, b, n, m, ns, c_feat, widths, round_out):
    _sa_check(cuda_dev, mlp.mlp_sa_fact2, mlp.sa_fact2_fits, b, n, m, ns, c_feat, widths, round_out,
              reserve=120 * round_out, seed=b + m + ns)


@pytest.mark.parametrize("ns,c_feat,widths", [(16, 96, (64, 64, 128)), (32, 6, (32, 48, 112))])
def test_sa_fact2_column_slice_within_f64_bound(cuda_dev, ns, c_feat, widths):
    _sa_check(cuda_dev, mlp.mlp_sa_fact2, mlp.sa_fact2_fits, 2, 1000, 300, ns, c_feat, widths, True, seed=5 + ns,
              slice_=True)


@pytest.mark.parametrize("b,n,m,ns,c_feat,widths", [
    (32, 1024, 512, 16, 64, (128, 196, 256)),   # SA3 at 32 frames
    (32, 1024, 512, 32, 64, (128, 196, 256)),
    (32, 512, 128, 16, 256, (256, 256, 512)),   # SA4
    (32, 512, 128, 32, 256, (256, 384, 512)),
    (3, 700, 129, 16, 64, (128, 196, 256)),     # a ragged last tile
    (3, 700, 129, 32, 256, (256, 384, 512)),
    (2, 1024, 300, 16, 64, (64, 144, 144)),     # a ragged last layer-3 block (16 of 128 columns), layer-2 n_pad 144
    (2, 1024, 300, 32, 64, (96, 208, 400)),     # n3 400: four layer-3 blocks, the last 16 wide; layer-2 n_pad 208
    (2, 1024, 300, 32, 64, (160, 144, 256)),    # layer-2 K 160
])
@pytest.mark.parametrize("round_out", [False, True])
def test_sa_fact2w_within_f64_bound(cuda_dev, b, n, m, ns, c_feat, widths, round_out):
    _sa_check(cuda_dev, mlp.mlp_sa_fact2w, mlp.sa_fact2w_fits, b, n, m, ns, c_feat, widths, round_out,
              reserve=120 * round_out, seed=b + m + ns + widths[2])


@pytest.mark.parametrize("ns,widths", [(16, (64, 144, 144)), (32, (256, 384, 512))])
def test_sa_fact2w_column_slice_within_f64_bound(cuda_dev, ns, widths):
    """the ragged last layer-3 block's MMA covers W3 rows past n3_pad: the store must stop at the layer's columns"""
    _sa_check(cuda_dev, mlp.mlp_sa_fact2w, mlp.sa_fact2w_fits, 2, 1000, 300, ns, 64, widths, True, seed=11 + ns,
              slice_=True)


def _sa_mutation(name, u, v, idx, n, l2, l3):
    """a reference that is wrong the way a kernel could be"""
    rows_u, rows_v = _sa_rows(idx, n, idx.size(1))
    w3, b3 = l3.w.clone(), l3.bias.clone()
    if name == "last_k3_chunk_dropped":
        k0 = (l2.n - 1) // 32 * 32
        w3[:, k0:] = 0
    elif name == "b3_rolled":
        b3[:l3.n] = b3[:l3.n].roll(1)
    elif name == "centre_from_previous_frame":
        ns = idx.size(2)
        m = idx.size(1)
        rows_u = rows_u.clone()
        rows_u[m * ns:(m + 1) * ns] -= n              # frame 1, centre 0: the same indices in frame 0
    return fb.sa_scale(u, v, rows_u, rows_v, l2.w, l2.bias, w3, b3, idx.size(2), False)


@pytest.mark.parametrize("fused,fits,c_feat,widths", [
    (mlp.mlp_sa_fact2, mlp.sa_fact2_fits, 96, (64, 96, 128)),
    (mlp.mlp_sa_fact2w, mlp.sa_fact2w_fits, 64, (128, 196, 256)),
], ids=["sa_fact2", "sa_fact2w"])
def test_sa_bound_catches_wrong_references(cuda_dev, fused, fits, c_feat, widths):
    b, n, m, ns = 2, 1024, 256, 32
    u, v, idx, l2, l3 = _factored_scale(cuda_dev, b, n, m, ns, c_feat, widths, seed=21)
    assert fits(l2, l3, ns)
    got = fused(u, v, idx, n, l2, l3)
    fb.check(got, *_sa_ref(u, v, idx, n, l2, l3, False), "correct reference")
    for name in ("last_k3_chunk_dropped", "b3_rolled", "centre_from_previous_frame"):
        with pytest.raises(AssertionError, match="outside the bound"):
            fb.check(got, *_sa_mutation(name, u, v, idx, n, l2, l3), name)


# ---- FP2-FP4: interpolation + two layers ----------------------------------------------------------------------------


def _nn_rows(nn_idx, m):
    b = nn_idx.size(0)
    return (torch.arange(b, device=nn_idx.device)[:, None, None] * m + nn_idx.long()).reshape(-1, 3)


def _fp_ref(known, skip, nn_idx, nn_w, c1, l1, l2, round_out, swap_w=False, skip_shift=0):
    m, c2 = known.size(1), known.size(2)
    w = nn_w.reshape(-1, 3)
    if swap_w:
        w = w[:, [1, 0, 2]]
    sk = skip if not skip_shift else skip.roll(skip_shift, dims=1)
    return fb.fp_module(known.reshape(-1, c2), _nn_rows(nn_idx, m), w, sk, c1, l1.w, l1.bias, l2.w, l2.bias, round_out)


@pytest.mark.parametrize("b,n,m,c2,c1,n1,n2", [
    (32, 512, 128, 1024, 512, 512, 512),     # FP4 at 32 frames
    (32, 1024, 512, 512, 256, 512, 512),     # FP3
    (32, 2048, 1024, 512, 96, 256, 256),     # FP2
    (3, 1000, 257, 1024, 512, 512, 512),     # the same three at 3 frames, a ragged last tile
    (3, 1000, 257, 512, 256, 512, 512),
    (3, 1000, 257, 512, 96, 256, 256),
    (3, 700, 129, 80, 52, 256, 384),         # a K chunk across the interpolated / skip columns; three layer-2 blocks
    (2, 640, 200, 512, 96, 256, 128),        # one layer-2 block
])
@pytest.mark.parametrize("round_out,reserve", [(False, 0), (True, 120)])
def test_fp2_within_f64_bound(cuda_dev, b, n, m, c2, c1, n1, n2, round_out, reserve):
    known, skip, nn_idx, nn_w, lds, l1, l2 = _fp_module(cuda_dev, b, n, m, c2, c1, n1, n2, seed=b + n + c2 + n2)
    assert mlp.fp2_fits(l1, l2)
    got = mlp.mlp_fp2(known, nn_idx, nn_w, skip.data_ptr(), lds, c1, l1, l2, round_out=round_out, reserve=reserve)
    fb.check(got, *_fp_ref(known, skip, nn_idx, nn_w, c1, l1, l2, round_out), f"fp2 b{b} n{n} {c2}+{c1}->{n1}->{n2}")


def test_fp2_unaligned_skip_rows_within_f64_bound(cuda_dev):
    """lds 97: skip rows only 4-byte aligned, every skip chunk on the generic producer path"""
    known, skip, nn_idx, nn_w, lds, l1, l2 = _fp_module(cuda_dev, 2, 640, 200, 512, 96, 256, 256, seed=5, lds=97)
    assert mlp.fp2_fits(l1, l2)
    got = mlp.mlp_fp2(known, nn_idx, nn_w, skip.data_ptr(), lds, 96, l1, l2, round_out=True)
    fb.check(got, *_fp_ref(known, skip, nn_idx, nn_w, 96, l1, l2, True), "fp2 lds 97")


def test_fp2_column_slice_within_f64_bound(cuda_dev):
    b, n, m, c2, c1 = 2, 1000, 300, 512, 256
    known, skip, nn_idx, nn_w, lds, l1, l2 = _fp_module(cuda_dev, b, n, m, c2, c1, 512, 384, seed=17)
    assert mlp.fp2_fits(l1, l2)
    ld, col0 = l2.n_pad + 136, 64
    out = torch.full((b * n, ld), -7.0, device=cuda_dev)
    mlp.mlp_fp2(known, nn_idx, nn_w, skip.data_ptr(), lds, c1, l1, l2, out=out, col0=col0)
    fb.check(out[:, col0:col0 + l2.n_pad], *_fp_ref(known, skip, nn_idx, nn_w, c1, l1, l2, False), "fp2 slice")
    assert bool((out[:, :col0] == -7.0).all()) and bool((out[:, col0 + l2.n_pad:] == -7.0).all())


def test_fp2_bound_catches_wrong_references(cuda_dev):
    known, skip, nn_idx, nn_w, lds, l1, l2 = _fp_module(cuda_dev, 2, 700, 129, 80, 52, 256, 384, seed=23, lds=60)
    got = mlp.mlp_fp2(known, nn_idx, nn_w, skip.data_ptr(), lds, 52, l1, l2)
    fb.check(got, *_fp_ref(known, skip, nn_idx, nn_w, 52, l1, l2, False), "correct reference")
    with pytest.raises(AssertionError, match="outside the bound"):
        fb.check(got, *_fp_ref(known, skip, nn_idx, nn_w, 52, l1, l2, False, swap_w=True), "weights 1 and 2 swapped")
    with pytest.raises(AssertionError, match="outside the bound"):
        fb.check(got, *_fp_ref(known, skip, nn_idx, nn_w, 52, l1, l2, False, skip_shift=4), "skip shifted by 4")


# ---- FP1: skip term + second layer ----------------------------------------------------------------------------------


def _fp1_ref(p, table, nn_idx, nn_w, m, ls, l2, round_out, bs=None):
    return fb.fp1_module(p, _nn_rows(nn_idx, m), nn_w.reshape(-1, 3), table, ls.w, ls.bias if bs is None else bs, l2.w,
                         l2.bias, round_out)


def _cn_rows(x, b, n):
    """[b, C, n] channel-major -> [b * n, C] point-major"""
    return x.transpose(1, 2).reshape(b * n, -1)


@pytest.mark.parametrize("b,n,m", [
    (32, 12288, 2048),   # the production shape
    (3, 1000, 333),      # frames end inside 64-row tiles
    (3, 1001, 333),      # n % 8 != 0
    (2, 77, 40),
    (5, 40, 17),         # every tile spans frames
])
def test_fp_fact2_within_f64_bound(cuda_dev, b, n, m):
    p, table, nn_idx, nn_w, ls, l2 = _fp1_module(cuda_dev, b, n, m, seed=b + n + m)
    assert mlp.fp_fact2_fits(ls, l2)
    assert torch.equal(table, mlp.tf32_round(table))            # the factor table is TF32 already: an exact operand
    got = mlp.mlp_fp_fact2(p, table, nn_idx, nn_w, m, ls, l2)
    assert got.shape == (b, 128, n)
    fb.check(_cn_rows(got, b, n), *_fp1_ref(p, table, nn_idx, nn_w, m, ls, l2, False), f"fp_fact2 b{b} n{n}")


@pytest.mark.parametrize("b,n,m", [(32, 12288, 2048), (3, 1001, 333), (5, 40, 17)])
def test_fp_fact2_rows_within_f64_bound(cuda_dev, b, n, m):
    p, table, nn_idx, nn_w, ls, l2 = _fp1_module(cuda_dev, b, n, m, seed=b + n + m + 1)
    assert mlp.fp_fact2_fits(ls, l2)
    out = torch.full((b * n, 1280), -7.25, device=cuda_dev)
    mlp.mlp_fp_fact2_rows(p, table, nn_idx, nn_w, m, ls, l2, out, 128, reserve=120 * (b == 32))
    fb.check(out[:, 128:256], *_fp1_ref(p, table, nn_idx, nn_w, m, ls, l2, True), f"fp_fact2_rows b{b} n{n}")
    assert bool((out[:, :128] == -7.25).all()) and bool((out[:, 256:] == -7.25).all())


def test_fp1_bound_catches_wrong_references(cuda_dev):
    b, n, m = 3, 1001, 333
    p, table, nn_idx, nn_w, ls, l2 = _fp1_module(cuda_dev, b, n, m, seed=29)
    got = _cn_rows(mlp.mlp_fp_fact2(p, table, nn_idx, nn_w, m, ls, l2), b, n)
    ref, bound = _fp1_ref(p, table, nn_idx, nn_w, m, ls, l2, False)
    fb.check(got, ref, bound, "correct reference")
    with pytest.raises(AssertionError, match="outside the bound"):
        fb.check(got, *_fp1_ref(p, table, nn_idx, nn_w, m, ls, l2, False, bs=torch.zeros_like(ls.bias)), "b_s omitted")
    rolled = [x.view(b, n, -1).roll(1, 0).reshape(b * n, -1) for x in (ref, bound)]
    with pytest.raises(AssertionError, match="outside the bound"):
        fb.check(got, *rolled, "frames rolled by one")
