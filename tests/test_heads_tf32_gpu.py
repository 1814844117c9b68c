"""The TF32 forms of the two DenseFusion launches that have no plain-layer twin, against float64 references of their
own operations (tests/f64_bounds.py), and FusedHeads on every routing path of run() against the float64 module graph:

  * pvn3d_mlp_dense_sum32 (conv4's 32-row sums of relu(A . W^T + b)): TF32 operands -> the reference is exact; within
    1e-5 of the 32-row sum of |A| . |W|^T + |b|; partial and lone groups, a ragged 128-column block, A_TF32 on and off,
    a column slice, the same bits twice;
  * pvn3d_mlp_dense_frame_bias (each head's first layer with the per-frame bias): 1-5 frames of 128-2048 rows, a ragged
    128-column block, ROUND_OUT on and off, a visibly different bias per frame;
  * FusedHeads: the 32-row-sum and per-frame-bias fast paths, and their fallbacks, each frame's embeddings scaled by
    1 + f so that a frame mix-up is gross.
Each check is also shown to fail on references that are wrong in the ways a kernel could be."""
import copy

import pytest
import torch

import f64_bounds as fb
from pvn3d_b200 import heads, mlp
from pvn3d_b200._lib import call, ptr

from helpers import heads_inputs, heads_modules
from test_heads_bf16_gpu import _module_graph

pytestmark = pytest.mark.gpu

RELU, ROUND_OUT, A_TF32 = mlp.MLP_RELU, mlp.MLP_ROUND_OUT, mlp.MLP_A_TF32


def _operands(dev, rows, k, n, lda, seed, a_tf32):
    """A [rows, lda] with columns k.. NaN (they must read as zero), pre-rounded to TF32 when the kernel copies it
    as is (A_TF32); the layer [n, k] TF32"""
    g = torch.Generator().manual_seed(seed)
    layer = mlp.PackedLayer(torch.randn(n, k, generator=g) * k ** -0.5, torch.randn(n, generator=g) * 0.1)
    layer.w, layer.bias = layer.w.to(dev), layer.bias.to(dev)
    a = torch.full((rows, lda), float("nan"))
    x = torch.randn(rows, k, generator=g).abs()
    a[:, :k] = mlp.tf32_round(x) if a_tf32 else x
    return a.to(dev), layer


def _rows_ref(a, k, layer, bias):
    """relu(tf32(A) . W^T + bias) per row, float64, with its accumulation bound"""
    return fb.dense(mlp.tf32_round(a[:, :k].contiguous()), layer.w[:, :k], bias)


# ---- pvn3d_mlp_dense_sum32 ------------------------------------------------------------------------------------------


def _sum32(a, lda, k, layer, a_tf32, out, col0):
    call("pvn3d_mlp_dense_sum32", a.device, ptr(a), lda, k, a.size(0), ptr(layer.w), ptr(layer.bias), layer.k_pad,
         layer.n_pad, RELU | (A_TF32 if a_tf32 else 0), ptr(out), out.size(-1), col0)
    return out[:, col0:col0 + layer.n_pad]


@pytest.mark.parametrize("rows", [4096, 1000, 4097, 20])
@pytest.mark.parametrize("k,n,lda", [(512, 1024, 1280), (500, 144, 520)])    # conv4; a ragged block, K not a chunk multiple
@pytest.mark.parametrize("a_tf32", [True, False])
def test_dense_sum32_within_f64_bound(cuda_dev, rows, k, n, lda, a_tf32):
    a, layer = _operands(cuda_dev, rows, k, n, lda, seed=rows + n, a_tf32=a_tf32)
    ref, bound = fb.group_sum(*_rows_ref(a, k, layer, layer.bias), 32)
    groups = (rows + 31) // 32
    col0, ldo = 8, layer.n_pad + 16
    out = torch.full((groups, ldo), -7.25, device=cuda_dev)
    got = _sum32(a, lda, k, layer, a_tf32, out, col0)
    fb.check(got, ref, bound, f"sum32 rows {rows} n_pad {layer.n_pad} a_tf32={a_tf32}")
    assert bool((out[:, :col0] == -7.25).all()) and bool((out[:, col0 + layer.n_pad:] == -7.25).all())
    again = torch.full_like(out, -7.25)
    assert torch.equal(_sum32(a, lda, k, layer, a_tf32, again, col0), got)        # fixed summation order


def test_dense_sum32_bound_catches_wrong_references(cuda_dev):
    rows, k, lda = 1000, 512, 1280
    a, layer = _operands(cuda_dev, rows, k, 1024, lda, seed=31, a_tf32=True)
    got = _sum32(a, lda, k, layer, True, torch.empty((32, layer.n_pad), device=cuda_dev), 0)
    per_row = _rows_ref(a, k, layer, layer.bias)
    ref, bound = fb.group_sum(*per_row, 32)
    fb.check(got, ref, bound, "correct reference")
    dropped = ref.clone()
    dropped[-1] = 0                                                   # the 8-row last group left out
    with pytest.raises(AssertionError, match="outside the bound"):
        fb.check(got, dropped, bound, "last partial group dropped")
    shifted = fb.group_sum(*(x[1:] for x in per_row), 32)             # groups of rows 1..32, 33..64, ..
    with pytest.raises(AssertionError, match="outside the bound"):
        fb.check(got, *shifted, "groups offset by one row")


# ---- pvn3d_mlp_dense_frame_bias -------------------------------------------------------------------------------------


def _frame_bias_operands(dev, frames, rpf, n, seed):
    k, lda = 768, 1280
    a, layer = _operands(dev, frames * rpf, k, n, lda, seed=seed, a_tf32=True)
    g = torch.Generator().manual_seed(seed + 1)
    fbias = torch.randn(frames, layer.n_pad, generator=g) * 0.1 + 0.5 * torch.arange(frames)[:, None]
    return a, layer, fbias.to(dev)


def _frame_bias(a, layer, fbias, rpf, round_out):
    out = torch.empty((a.size(0), layer.n_pad), device=a.device)
    call("pvn3d_mlp_dense_frame_bias", a.device, ptr(a), a.size(1), 768, a.size(0), rpf, ptr(layer.w), ptr(fbias),
         layer.k_pad, layer.n_pad, RELU | A_TF32 | (ROUND_OUT if round_out else 0), ptr(out), out.size(-1), 0)
    return out


def _frame_bias_ref(a, layer, fbias, rpf, round_out):
    ref, bound = _rows_ref(a, 768, layer, fbias.repeat_interleave(rpf, 0))
    return fb.round_tf32(ref, bound) if round_out else (ref, bound)


@pytest.mark.parametrize("frames,rpf,n", [(1, 2048, 1024), (2, 1280, 144), (3, 128, 1024), (4, 1280, 1024), (5, 128, 144),
                                          (5, 2048, 144)])
@pytest.mark.parametrize("round_out", [True, False])
def test_dense_frame_bias_within_f64_bound(cuda_dev, frames, rpf, n, round_out):
    a, layer, fbias = _frame_bias_operands(cuda_dev, frames, rpf, n, seed=frames * rpf + n)
    got = _frame_bias(a, layer, fbias, rpf, round_out)
    fb.check(got, *_frame_bias_ref(a, layer, fbias, rpf, round_out),
             f"frame_bias {frames} x {rpf} n_pad {layer.n_pad} round_out={round_out}")


def test_dense_frame_bias_bound_catches_the_previous_frames_bias(cuda_dev):
    frames, rpf = 3, 1280
    a, layer, fbias = _frame_bias_operands(cuda_dev, frames, rpf, 1024, seed=37)
    got = _frame_bias(a, layer, fbias, rpf, True)
    fb.check(got, *_frame_bias_ref(a, layer, fbias, rpf, True), "correct reference")
    with pytest.raises(AssertionError, match="outside the bound"):
        fb.check(got, *_frame_bias_ref(a, layer, fbias.roll(1, 0), rpf, True), "frame f - 1's bias")


# ---- FusedHeads, one case per routing path of run() -----------------------------------------------------------------


@pytest.fixture(scope="module")
def modules(cuda_dev):
    mods = heads_modules()
    return [m.to(cuda_dev).eval() for m in mods], [copy.deepcopy(m).double().to(cuda_dev).eval() for m in mods]


@pytest.mark.parametrize("b,n", [
    (3, 1280),    # n % 128 == 0: 32-row sums and the per-frame bias
    (3, 1056),    # n % 32 == 0, n % 128 != 0: 32-row sums, one first-layer launch per frame
    (3, 1000),    # both fallbacks
])
def test_tf32_heads_routes_match_f64_module_graph(cuda_dev, modules, monkeypatch, b, n):
    mods32, mods64 = modules
    rgb_emb, cld_emb = heads_inputs(b, n)
    scale = (1.0 + torch.arange(b, dtype=torch.float32))[:, None, None]        # frame f x (1 + f): a mix-up is gross
    rgb_emb, cld_emb = (rgb_emb * scale).to(cuda_dev), (cld_emb * scale).to(cuda_dev)
    eng = heads.FusedHeads(*mods32, device=cuda_dev)
    launches = []
    orig = heads.call

    def spy(name, *args):
        launches.append(name)
        return orig(name, *args)

    monkeypatch.setattr(heads, "call", spy)
    got = eng(rgb_emb, cld_emb)
    monkeypatch.undo()
    # the route run() took: frame-bias launches only at n % 128 == 0, per-frame first layers and the per-point conv4
    # launch otherwise
    dense = 1 + (n % 32 != 0) + sum(len(hd.rest) + (0 if n % 128 == 0 else b) for hd in eng.heads)
    assert launches.count("pvn3d_mlp_dense_sum32") == 1
    assert launches.count("pvn3d_mlp_dense_frame_bias") == (3 if n % 128 == 0 else 0)
    assert launches.count("pvn3d_mlp_dense") == dense, launches
    with torch.no_grad():
        want = _module_graph(mods64, rgb_emb.double(), cld_emb.double())
    for name, g, w in zip(("kp_of", "seg", "ctr_of"), got, want):
        assert g.dtype == torch.float32 and g.shape == w.shape, name
        for f in range(b):
            gf, wf = g[f].double(), w[f]
            s = float(wf.abs().mean())
            err = (gf - wf).abs()
            print(f"{name} [{b}x{n}] frame {f}: mean {float(err.mean()) / s:.2e} max {float(err.max()) / s:.2e}")
            # the TF32 class of tests/test_heads_gpu.py, per frame
            assert float(err.mean()) <= 3e-3 * s and float(err.max()) <= 3e-2 * s, (name, f)
