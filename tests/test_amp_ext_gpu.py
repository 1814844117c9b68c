"""The float16 / bfloat16 forms of group_points, three_interpolate, their grads and the PSPNet backward (the pvn3d_*_16
entry points of csrc/pn2_ops.cu and csrc/determinism.cu, reached through pvn3d_b200._ext and .deterministic) at the
training shapes of test_deterministic_gpu.py (24 frames x 12288 points, device FPS / ball query / three_nn plans):

  * group_points is a copy: bit-equal to torch.gather of the 16-bit features;
  * three_interpolate is bit-equal to round16(the float32 kernel on the widened features);
  * the ordered grads are bit-equal to round16(determinism_ref's float32 restatement on the widened gradient), and
    repeat bit for bit across calls and streams; the PSP backward likewise on the POOLS / UPS cases;
  * the atomic grads are within grad_ref's float32 bound plus half a 16-bit ulp of the float64 sum;
  * float16 overflow gives inf, NaN propagates, out-of-range indices contribute nothing, no host sync.
"""
import types

import numpy as np
import pytest
import torch

import determinism_ref as dr
import grad_ref as gr
from helpers import SA_LEVELS
from pvn3d_b200 import _ext, deterministic, synth
from test_deterministic_gpu import POOLS, UPS

pytestmark = pytest.mark.gpu

B, N = 24, 12288
SA_C = (6, 96, 256, 512)
FP_C = (256, 512, 512, 1024)
DTYPES = [torch.bfloat16, torch.float16]
DT_IDS = ["bf16", "fp16"]


@pytest.fixture
def det_on():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


def _weights(d2):
    recip = 1.0 / (torch.sqrt(d2) + 1e-8)
    return (recip / recip.sum(2, keepdim=True)).contiguous()


@pytest.fixture(scope="module")
def plan(cuda_dev):
    frames = synth.make_batch("ycb", B, n_points=N, config_id=31)
    xyz = torch.from_numpy(np.stack([f.pcld for f in frames])).to(cuda_dev).contiguous()
    levels, fps = [xyz], []
    for _, m, _, _ in SA_LEVELS:
        idx = _ext.furthest_point_sampling(levels[-1], m)
        fps.append(idx)
        levels.append(_ext.gather_xyz(levels[-1], idx))
    balls = {(li, ns): _ext.ball_query(levels[li + 1], levels[li], r, ns)
             for li, (_, _, radii, nss) in enumerate(SA_LEVELS) for r, ns in zip(radii, nss)}
    nn = {lu: (lambda d2, i: (i, _weights(d2)))(*_ext.three_nn(levels[lu], levels[lu + 1])) for lu in range(4)}
    return types.SimpleNamespace(levels=levels, fps=fps, balls=balls, nn=nn)


def _randn(shape, dev, seed, dtype):
    return torch.randn(shape, generator=torch.Generator(device=dev).manual_seed(seed), device=dev).to(dtype)


def _bits16(x):
    return x.contiguous().view(torch.int16)


def _check_bits16(got, want, what):
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype)
    if not torch.equal(_bits16(got), _bits16(want)):
        raise AssertionError(f"{what}: {int((_bits16(got) != _bits16(want)).sum())} elements differ in bits")


def half_ulp16(v: torch.Tensor, dtype) -> torch.Tensor:
    """half the spacing of `dtype` at |v| (float64): 2^(e - p) / 2 with e = floor(log2 |v|) clamped to the normal range"""
    p, emin = (10, -14) if dtype == torch.float16 else (7, -126)
    _, ex = torch.frexp(v.double().abs())
    e = torch.clamp(ex.long() - 1, min=emin)
    return torch.ldexp(torch.full_like(v, 0.5, dtype=torch.float64), e - p)


def check_atomic16(got, r: gr.Ref, what):
    """|got - ref| <= gamma_k sum|t| + half a 16-bit ulp of got; k = 0 gives +0.0"""
    err = (got.double() - r.ref).abs()
    bound = r.bound() + half_ulp16(got, got.dtype)
    bad = ~(err <= bound)
    bad |= (r.k.expand_as(r.ref) == 0) & (_bits16(got) != 0)
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the bound"
    print(f"{what}: worst |got - ref| / bound {float((err / bound).max()):.3g}")


# ---- forward --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("ns_i", [0, 1])
@pytest.mark.parametrize("li", [0, 1, 2, 3])
def test_group_points_is_a_copy(cuda_dev, plan, li, ns_i, dtype):
    n, m, _, nss = SA_LEVELS[li]
    idx = plan.balls[(li, nss[ns_i])]
    feats = _randn((B, SA_C[li], n), cuda_dev, 10 * li + ns_i, dtype)
    got = _ext.group_points(feats, idx)
    want = feats.gather(2, idx.long().reshape(B, 1, -1).expand(-1, SA_C[li], -1)).reshape(got.shape)
    _check_bits16(got, want, f"group SA{li + 1} ns{nss[ns_i]}")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("lu", [0, 1, 2, 3])
def test_three_interpolate_is_round16_of_float32(cuda_dev, plan, lu, dtype):
    idx, w = plan.nn[lu]
    m = plan.levels[lu + 1].size(1)
    feats = _randn((B, FP_C[lu], m), cuda_dev, 40 + lu, dtype)
    got = _ext.three_interpolate(feats, idx, w)
    _check_bits16(got, _ext.three_interpolate(feats.float(), idx, w).to(dtype), f"interp FP{lu + 1}")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_odd_sizes_take_the_scalar_forms(cuda_dev, dtype):
    """an odd slot count / point count (one element per store) gives the same bits"""
    gen = torch.Generator(device=cuda_dev).manual_seed(50)
    feats = _randn((3, 7, 101), cuda_dev, 51, dtype)
    idx = torch.randint(0, 101, (3, 13, 5), generator=gen, device=cuda_dev, dtype=torch.int32)
    want = feats.gather(2, idx.long().reshape(3, 1, -1).expand(-1, 7, -1)).reshape(3, 7, 13, 5)
    _check_bits16(_ext.group_points(feats, idx), want, "group, odd slots")
    idx3 = torch.randint(0, 101, (3, 77, 3), generator=gen, device=cuda_dev, dtype=torch.int32)
    w = torch.rand((3, 77, 3), generator=gen, device=cuda_dev)
    _check_bits16(_ext.three_interpolate(feats, idx3, w), _ext.three_interpolate(feats.float(), idx3, w).to(dtype),
                  "interp, odd n")


# ---- grads ----------------------------------------------------------------------------------------------------------
def _both(fn, args):
    atomic = fn(*args)
    torch.use_deterministic_algorithms(True)
    try:
        ordered = fn(*args)
        again = fn(*args)
    finally:
        torch.use_deterministic_algorithms(False)
    _check_bits16(again, ordered, "ordered, second call")
    return atomic, ordered


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("ns_i", [0, 1])
@pytest.mark.parametrize("li", [0, 1, 2, 3])
def test_group_grad(cuda_dev, plan, li, ns_i, dtype):
    n, m, _, nss = SA_LEVELS[li]
    idx = plan.balls[(li, nss[ns_i])]
    g = _randn((B, SA_C[li], m, nss[ns_i]), cuda_dev, 100 + 10 * li + ns_i, dtype)
    atomic, ordered = _both(_ext.group_points_grad, (g, idx, n))
    what = f"group grad SA{li + 1} ns{nss[ns_i]} {dtype}"
    _check_bits16(ordered, dr.group_grad32(g.float(), idx, n).to(dtype), what)
    check_atomic16(atomic, gr.group_grad(g, idx, n), what + " atomic")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("lu", [0, 1, 2, 3])
def test_interp_grad(cuda_dev, plan, lu, dtype):
    idx, w = plan.nn[lu]
    n, m = plan.levels[lu].size(1), plan.levels[lu + 1].size(1)
    g = _randn((B, FP_C[lu], n), cuda_dev, 210 + lu, dtype)
    atomic, ordered = _both(_ext.three_interpolate_grad, (g, idx, w, m))
    what = f"interp grad FP{lu + 1} {dtype}"
    _check_bits16(ordered, dr.interp_grad32(g.float(), idx, w, m).to(dtype), what)
    check_atomic16(atomic, gr.interp_grad(g, idx, w, m), what + " atomic")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_out_of_range_indices_contribute_nothing(cuda_dev, det_on, dtype):
    b, c, n, j = 3, 37, 500, 4096
    gen = torch.Generator(device=cuda_dev).manual_seed(700)
    idx = torch.randint(-50, n + 50, (b, j), generator=gen, device=cuda_dev, dtype=torch.int32)
    idx[0, :7] = torch.tensor([-2 ** 31, 2 ** 31 - 1, n, -1, n - 1, 0, n + 1], dtype=torch.int32)
    g = _randn((b, c, j), cuda_dev, 701, dtype)
    w = torch.rand((b, j, 3), generator=gen, device=cuda_dev)
    idx3 = torch.randint(-5, n + 5, (b, j, 3), generator=gen, device=cuda_dev, dtype=torch.int32)
    _check_bits16(_ext.group_points_grad(g.reshape(b, c, j // 16, 16), idx.reshape(b, j // 16, 16), n),
                  dr.gather_grad32(g.float(), idx, n).to(dtype), "group, out-of-range")
    _check_bits16(_ext.three_interpolate_grad(g, idx3, w, n), dr.interp_grad32(g.float(), idx3, w, n).to(dtype),
                  "interp, out-of-range")


# ---- PSPNet pooling and upsampling ----------------------------------------------------------------------------------
def _pool_bwd(g, ih, iw):
    x = torch.zeros((g.size(0), g.size(1), ih, iw), dtype=g.dtype, device=g.device, requires_grad=True)
    deterministic.adaptive_avg_pool2d(x, tuple(g.shape[-2:])).backward(g)
    return x.grad


def _up_bwd(g, ih, iw, align, scale_factor=None):
    x = torch.zeros((g.size(0), g.size(1), ih, iw), dtype=g.dtype, device=g.device, requires_grad=True)
    size = None if scale_factor else tuple(g.shape[-2:])
    deterministic.interpolate(x, size=size, scale_factor=scale_factor, mode="bilinear", align_corners=align).backward(g)
    return x.grad


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("case", POOLS, ids=[f"{a}x{b}->{c}x{d}" for a, b, c, d in POOLS])
def test_pool_backward(cuda_dev, det_on, case, dtype):
    ih, iw, oh, ow = case
    g = _randn((2, 3, oh, ow), cuda_dev, 800 + ih, dtype)
    got = _pool_bwd(g, ih, iw)
    _check_bits16(got, dr.pool_backward32(g.float().reshape(6, oh, ow), ih, iw).reshape(got.shape).to(dtype),
                  f"pool {case}")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("case", UPS, ids=[f"{a}x{b}->{c}x{d}-{e}-{f}" for a, b, c, d, e, f in UPS])
def test_upsample_backward(cuda_dev, det_on, case, dtype):
    ih, iw, oh, ow, align, sf = case
    g = _randn((2, 2, oh, ow), cuda_dev, 900 + ih, dtype)
    got = _up_bwd(g, ih, iw, align, sf)
    want = dr.upsample_backward32(g.float().reshape(4, oh, ow), ih, iw, align, sf).reshape(got.shape).to(dtype)
    _check_bits16(got, want, f"upsample {case}")


# ---- inf, NaN -------------------------------------------------------------------------------------------------------
def test_fp16_overflow_is_inf_and_nan_propagates(cuda_dev, plan):
    h = torch.float16
    n, m, _, nss = SA_LEVELS[1]
    idx = torch.zeros((1, 4, 8), dtype=torch.int32, device=cuda_dev)           # 32 slots on point 0
    idx[0, 3] = 1                                                               # 8 slots on point 1
    g = torch.full((1, 2, 4, 8), 60000.0, dtype=h, device=cuda_dev)
    g[0, 1, 3, 5] = float("nan")
    for det in (False, True):
        torch.use_deterministic_algorithms(det)
        try:
            out = _ext.group_points_grad(g, idx, 3)
            gi = _ext.three_interpolate_grad(g.reshape(1, 2, 32), idx.reshape(1, 32, 1).expand(1, 32, 3).contiguous(),
                                             torch.full((1, 32, 3), 0.5, device=cuda_dev), 3)
            x = torch.zeros((1, 2, 6, 6), dtype=h, device=cuda_dev, requires_grad=True)
            deterministic.interpolate(x, size=(60, 80), mode="bilinear", align_corners=False).backward(
                torch.full((1, 2, 60, 80), 60000.0, dtype=h, device=cuda_dev))
        finally:
            torch.use_deterministic_algorithms(False)
        assert bool(torch.isinf(out[0, 0, :2]).all()) and bool((out[0, 0, :2] > 0).all()), (det, out)
        assert float(out[0, 0, 2]) == 0.0 and bool(torch.isnan(out[0, 1, 1])), (det, out)
        assert bool(torch.isinf(gi[0, 0, :2]).all()) and bool(torch.isnan(gi[0, 1, 1])), (det, gi)
        if det:                                     # the ordered PSP backward (torch's own runs with the switch off)
            assert bool(torch.isinf(x.grad).all()) and bool((x.grad > 0).all())
    feats = torch.full((1, 1, 4), 60000.0, dtype=h, device=cuda_dev)
    feats[0, 0, 3] = float("nan")
    i3 = torch.tensor([[[0, 1, 2], [0, 1, 3]]], dtype=torch.int32, device=cuda_dev)
    out = _ext.three_interpolate(feats, i3, torch.ones((1, 2, 3), device=cuda_dev))
    assert bool(torch.isinf(out[0, 0, 0])) and bool(torch.isnan(out[0, 0, 1])), out
    assert bool(torch.isnan(_ext.group_points(feats, i3[:, :, 2:3].contiguous())[0, 0, 1, 0]))


# ---- determinism, streams, syncs ------------------------------------------------------------------------------------
def _step(plan, dev, dtype):
    n, m, _, nss = SA_LEVELS[1]
    gg = _randn((B, SA_C[1], m, nss[1]), dev, 1200, dtype)
    gi = _randn((B, 64, n), dev, 1201, dtype)
    gp = _randn((B, 32, 6, 6), dev, 1203, dtype)
    gu = _randn((B, 32, 60, 80), dev, 1204, dtype)
    feats = _randn((B, SA_C[1], n), dev, 1205, dtype)
    idx, w = plan.nn[1]
    ball = plan.balls[(1, nss[1])]
    return lambda: [_ext.group_points_grad(gg, ball, n), _ext.three_interpolate_grad(gi, idx, w, m),
                    _pool_bwd(gp, 60, 80), _up_bwd(gu, 6, 6, False), _ext.group_points(feats, ball),
                    _ext.three_interpolate(feats[:, :, :m].contiguous(), idx, w)]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_two_calls_and_two_streams_give_the_same_bits(cuda_dev, plan, det_on, dtype):
    run = _step(plan, cuda_dev, dtype)
    first, second = run(), run()
    side = torch.cuda.Stream(cuda_dev)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        third = run()
    fourth = run()
    torch.cuda.synchronize()
    for i, (a, *others) in enumerate(zip(first, second, third, fourth)):
        assert a.dtype == dtype, i
        for o in others:
            assert torch.equal(_bits16(a), _bits16(o)), i


@pytest.mark.parametrize("det", [False, True], ids=["atomic", "deterministic"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_16_bit_calls_make_no_host_sync(cuda_dev, plan, dtype, det):
    run = _step(plan, cuda_dev, dtype)
    torch.use_deterministic_algorithms(det)
    try:
        run()
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            run()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    finally:
        torch.use_deterministic_algorithms(False)
    torch.cuda.synchronize()
