"""pvn3d_psp_tail_rows on the device: the CNN's up_3 + final at the sampled pixels.

  * the kernel against the float64 reference of its own operation (cnn_tail.sampled_tail_reference) with the
    element-wise bounds of tests/f64_bounds.py, f32 (TF32-rounded) rows and bf16 rows, and the same check shown to fail
    against references that are wrong the way the kernel could be;
  * FusedPVN3D on a CNN with the reference's layout: the sampled path is taken, and its outputs agree with the dense path;
  * compat.patch_pvn3d_forward rebuilds the engine when the tail's weights change;
  * with the staged reference Python: the reference's own Modified_PSPNet is recognised and agrees.
"""
import copy

import pytest
import torch
import torch.nn.functional as F

import f64_bounds as fb
from cnn_tail_cases import SIZES, border_choose, half_map
from helpers import load_reference_python
from network_cases import network_inputs
from pvn3d_b200 import compat, network, testing
from pvn3d_b200.cnn_tail import PspTail, sampled_tail_reference
from pvn3d_b200.heads import FusedHeads
from pvn3d_b200.mlp import tf32_round

pytestmark = pytest.mark.gpu

BILINEAR = 2.0 ** -21   # the fp32 weights and fma chain of a bilinear sample, relative to sum |weight * value|
BF16_ROUND = 2.0 ** -7  # two bf16 roundings of nearby values: one bf16 ulp relative to the rounded value


@pytest.fixture(autouse=True)
def _fp32_reference():
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _tail(dev, prelu_params=64, seed=3):
    return PspTail.from_cnn(testing.StandInPSPNet(seed=seed, prelu_params=prelu_params).to(dev))


def _packed(tail):
    """the weights the kernel multiplies: TF32-rounded, as packed"""
    return tail.layer1.w, tail.layer1.bias, tail.slope, tail.layer2.w, tail.layer2.bias


def _layers(taps, e_taps, packed, bf16):
    """(reference rows, bound) from float64 taps and their uncertainty: both layers with every rounding of the kernel"""
    w1, b1, slope, w2, b2 = packed
    a, e = fb.round_tf32(taps, e_taps)
    v, e = fb.dense(a, w1, b1, e, relu=False)
    s = slope.double()
    h = torch.where(v >= 0, v, s * v)
    h, e = fb.round_tf32(h, e * s.abs().clamp_min(1.0) + fb.F32 * h.abs())       # PReLU: max(1, |slope|)-Lipschitz
    y, e = fb.dense(h, w2, b2, e, relu=False)
    if bf16:
        r = y.float().to(torch.bfloat16).double()
        return r, e + BF16_ROUND * r.abs()
    return fb.round_tf32(y, e)


def _reference(tail, x_half, choose, bf16=False, taps_edit=None):
    _, _, taps = sampled_tail_reference(x_half, choose, _packed(tail), taps_round=taps_edit)
    _, _, taps_abs = sampled_tail_reference(x_half.abs(), choose, _packed(tail))
    return _layers(taps, BILINEAR * taps_abs, _packed(tail), bf16)


def _run(tail, x_half, choose, bf16=False, ldo=128, col0=0):
    out = torch.full((choose.size(0) * choose.size(2), ldo), -7.25, device=x_half.device,
                     dtype=torch.bfloat16 if bf16 else torch.float32)
    tail.rows(x_half, choose, out, col0)
    return out


@pytest.mark.parametrize("bf16", [False, True], ids=["tf32", "bf16"])
@pytest.mark.parametrize("b", [1, 3])
@pytest.mark.parametrize("h,w", SIZES)
def test_rows_within_the_float64_bound(cuda_dev, h, w, b, bf16):
    tail = _tail(cuda_dev)
    n = 300                                              # not a multiple of the 128-row tile; b = 3: tiles span two frames
    x = half_map(b, h, w, seed=h + b).to(cuda_dev)
    choose = border_choose(b, n, 2 * h, 2 * w, seed=w).to(cuda_dev)
    got = _run(tail, x, choose, bf16)
    ref, bound = _reference(tail, x, choose, bf16)
    fb.check(got, ref, bound, f"psp_tail {b}x{n} of {2 * h}x{2 * w} {'bf16' if bf16 else 'tf32'}")
    if not bf16:
        assert torch.equal(got, tf32_round(got))         # the rows are TF32 values


def test_single_slope_prelu_and_a_column_slice(cuda_dev):
    tail = _tail(cuda_dev, prelu_params=1)
    b, h, w, n = 2, 30, 41, 515
    x = half_map(b, h, w, seed=9).to(cuda_dev)
    choose = border_choose(b, n, 2 * h, 2 * w, seed=4).to(cuda_dev)
    for bf16 in (False, True):
        got = _run(tail, x, choose, bf16, ldo=1280, col0=256)
        ref, bound = _reference(tail, x, choose, bf16)
        fb.check(got[:, 256:384], ref, bound, "psp_tail into columns 256..383")
        assert bool((got[:, :256] == -7.25).all()) and bool((got[:, 384:] == -7.25).all())


def _module_rows(tail, x, choose, align_corners=True, pad_mode="constant"):
    """final(up_3(x)) at the sampled pixels through torch's own float64 ops, with the packed weights"""
    w1, b1, slope, w2, b2 = (t.double() for t in _packed(tail))
    up = F.interpolate(x.double(), scale_factor=2, mode="bilinear", align_corners=align_corners)
    kernel = w1.view(64, 3, 3, 64).permute(0, 3, 1, 2)
    v = F.conv2d(F.pad(up, (1, 1, 1, 1), mode=pad_mode), kernel, b1)
    y = F.conv2d(F.prelu(v, slope), w2.view(128, 64, 1, 1), b2)
    bsz, n = choose.size(0), choose.size(2)
    return torch.gather(y.flatten(2), 2, choose.repeat(1, 128, 1)).transpose(1, 2).reshape(bsz * n, 128)


def _swap_dy_dx(taps):
    return taps.view(-1, 3, 3, 64).transpose(1, 2).reshape(taps.shape)


def _drop_tap(taps):
    t = taps.clone().view(-1, 9, 64)
    t[:, 5] = 0
    return t.view(taps.shape)


WRONG = ["one tap dropped", "taps transposed", "align_corners=False", "border taps clamped", "neighbour frame's map",
         "slope of the wrong channel"]


@pytest.mark.parametrize("what", WRONG)
def test_the_bound_rejects_a_wrong_reference(cuda_dev, what):
    tail = _tail(cuda_dev)
    b, h, w, n = 3, 30, 41, 300
    x = half_map(b, h, w, seed=2).to(cuda_dev)
    choose = border_choose(b, n, 2 * h, 2 * w, seed=6).to(cuda_dev)
    got = _run(tail, x, choose)
    ref, bound = _reference(tail, x, choose)
    fb.check(got, ref, bound, "the right reference")
    fb.check(_module_rows(tail, x, choose), ref, bound, "torch's own float64 ops")
    if what == "one tap dropped":
        wrong, _ = _reference(tail, x, choose, taps_edit=_drop_tap)
    elif what == "taps transposed":
        wrong, _ = _reference(tail, x, choose, taps_edit=_swap_dy_dx)
    elif what == "align_corners=False":
        wrong = _module_rows(tail, x, choose, align_corners=False)
    elif what == "border taps clamped":
        wrong = _module_rows(tail, x, choose, pad_mode="replicate")
    elif what == "neighbour frame's map":
        wrong, _ = _reference(tail, x.roll(1, 0), choose)
    else:
        other = _tail(cuda_dev)
        other.slope = tail.slope.roll(1)
        wrong, _ = _reference(other, x, choose)
    with pytest.raises(AssertionError, match="outside the bound"):
        fb.check(got, wrong, bound, what)


def test_out_of_range_index_gives_a_nan_row(cuda_dev):
    tail = _tail(cuda_dev)
    b, h, w, n = 2, 30, 41, 300
    x = half_map(b, h, w, seed=5).to(cuda_dev)
    choose = border_choose(b, n, 2 * h, 2 * w, seed=8).to(cuda_dev)
    bad = choose.clone()
    bad[0, 0, 7], bad[1, 0, 130], bad[1, 0, 299] = 4 * h * w, -1, 2 ** 40
    rows = [7, n + 130, n + 299]
    keep = torch.ones(b * n, dtype=torch.bool, device=cuda_dev)
    keep[rows] = False
    for bf16 in (False, True):
        got, want = _run(tail, x, bad, bf16), _run(tail, x, choose, bf16)
        assert bool(got[rows].isnan().all())
        assert torch.equal(got[keep], want[keep])


# ---- the engine ------------------------------------------------------------------------------------------------------


class _Opaque(torch.nn.Module):
    """the same CNN behind a wrapper whose layout PspTail.from_cnn does not recognise: the dense path"""

    def __init__(self, inner):
        super().__init__()
        self.inner = inner

    def forward(self, x):
        return self.inner(x)


def _model(n, dev, seed=5):
    m = testing.StandInPVN3D(n, seed=seed)
    m.cnn = testing.StandInPSPNet(seed=seed, prelu_params=64)
    return m.to(dev).eval()


def _dense_twin(m):
    twin = copy.copy(m)
    twin._modules = dict(m._modules, cnn=_Opaque(m.cnn))
    return twin


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_engine_takes_the_sampled_path_and_agrees_with_the_dense_one(cuda_dev, precision):
    b, n = 2, 4096
    m = _model(n, cuda_dev)
    pc, rgb, choose = (t.to(cuda_dev) for t in network_inputs(b, n))
    net = network.FusedPVN3D(m, cuda_dev, precision)
    dense_net = network.FusedPVN3D(_dense_twin(m), cuda_dev, precision)
    assert net.tail is not None and dense_net.tail is None
    calls, tables = [], []
    hooks = [m.cnn.final.register_forward_hook(lambda *a: calls.append("final")),
             m.cnn.up_3.register_forward_hook(lambda *a: calls.append("up_3"))]
    run = net.heads.run
    net.heads.run = lambda x, *a: (tables.append(x[:, FusedHeads.RGB_COL0:FusedHeads.RGB_COL0 + 128].clone()), run(x, *a))[1]
    autocast = torch.autocast("cuda", dtype=torch.bfloat16, enabled=precision == "bf16")
    with torch.no_grad(), autocast:
        got = net(pc, rgb, choose)
        assert calls == []                                 # neither up_3 nor final ran
        for hk in hooks:
            hk.remove()
        want = dense_net(pc, rgb, choose)
        x_half = net.tail.trunk(rgb)
    assert x_half.dtype == (torch.bfloat16 if precision == "bf16" else torch.float32)
    direct = _run(net.tail, x_half, choose, bf16=precision == "bf16")
    assert torch.equal(tables[0], direct)
    mean_tol, max_tol = (3e-3, 3e-2) if precision == "tf32" else (2e-2, 2e-1)
    for name, g, w_ in zip(("kp_of", "seg", "ctr_of"), got, want):
        assert g.shape == w_.shape and g.dtype == torch.float32, name
        scale, err = float(w_.abs().max()), (g - w_).abs()
        print(f"{name} [{precision}]: sampled vs dense mean {float(err.mean()) / scale:.2e} max {float(err.max()) / scale:.2e}")
        assert float(err.mean()) <= mean_tol * scale and float(err.max()) <= max_tol * scale, name


def test_patch_rebuilds_the_engine_when_the_tail_weights_change(cuda_dev):
    b, n = 1, 4096
    cls = type("PatchedStandIn", (testing.StandInPVN3D,), {})
    compat.patch_pvn3d_forward(cls)
    m = cls.__new__(cls)
    m.__dict__.update(_model(n, cuda_dev).__dict__)
    x = [t.to(cuda_dev) for t in network_inputs(b, n)]
    with torch.no_grad():
        before = m(*x)
        eng = compat.fused_engine(m, cuda_dev)
        assert eng.tail is not None and compat.fused_engine(m, cuda_dev) is eng
        m.cnn.final[0].weight.mul_(1.5)
        after = m(*x)
        assert compat.fused_engine(m, cuda_dev) is not eng
        want = network.FusedPVN3D(m, cuda_dev)(*x)
    assert all(torch.equal(g, w_) for g, w_ in zip(after, want))
    assert not torch.equal(after[1], before[1])


def test_reference_pspnet_is_recognised_and_agrees(cuda_dev):
    if load_reference_python() is None:
        pytest.skip("the reference Python is not staged under oracle/_ref/py")
    from lib.pspnet import Modified_PSPNet

    torch.manual_seed(11)
    cnn = Modified_PSPNet(sizes=(1, 2, 3, 6), psp_size=512, deep_features_size=256, backend="resnet34", pretrained=False)
    testing.randomize_bn_(cnn, 12)
    cnn = cnn.to(cuda_dev).eval()
    wrapper = torch.nn.Module()
    wrapper.model = cnn
    tail = PspTail.from_cnn(wrapper)
    assert tail is not None and tail.model is cnn
    b, n, hh, ww = 2, 1000, 120, 160
    rgb = torch.rand(b, 3, hh, ww, generator=torch.Generator().manual_seed(1)).to(cuda_dev)
    choose = border_choose(b, n, hh, ww, seed=2).to(cuda_dev)
    with torch.no_grad():
        emb, _ = cnn(rgb)
        x_half = tail.trunk(rgb)
    assert emb.shape == (b, 128, hh, ww) and x_half.shape == (b, 64, hh // 2, ww // 2)
    got = _run(tail, x_half, choose)
    ref, bound = _reference(tail, x_half, choose)
    fb.check(got, ref, bound, "reference Modified_PSPNet tail")
    # torch's fp32 graph: unrounded weights and operands, so TF32-class agreement over the rows' scale
    dense = torch.gather(emb.flatten(2), 2, choose.repeat(1, 128, 1)).transpose(1, 2).reshape(b * n, 128)
    err, scale = (got - dense).abs(), float(dense.abs().max())
    print(f"sampled vs torch fp32 dense: mean {float(err.mean()) / scale:.2e} max {float(err.max()) / scale:.2e}")
    assert float(err.mean()) <= 1e-3 * scale and float(err.max()) <= 1e-2 * scale
