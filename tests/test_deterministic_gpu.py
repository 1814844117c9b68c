"""The fixed-order backward of torch.use_deterministic_algorithms(True) (csrc/determinism.cu, pvn3d_b200.deterministic,
the routing in pvn3d_b200._ext) against the float32 restatements and float64 adjoints of tests/determinism_ref.py:

  * the three PointNet++ grads at 24 frames x 12288 points (device FPS / ball query / three_nn plans, as
    test_pn2_grad_f64_gpu.py builds them): bit-equal to the restatement, within grad_ref's float64 bound, within twice
    that bound of today's atomic path; edge cases (empty balls, one or two known points, out-of-range indices, past
    2^31, empty shapes, the batch limit);
  * adaptive_avg_pool2d / upsample_bilinear2d backward at the PSPNet shapes and odd sizes: bit-equal to the
    restatement, within the float64 bound, bit-equal to torch's own backward where each input element gets one term;
    the restatement's taps against torch's forward on one-hot inputs;
  * repeat bits, two streams, no host sync; mode off launches exactly what it launched before;
  * one training step of the staged reference PVN3D, twice, in a subprocess under deterministic mode: bit-equal
    parameter gradients, and torch's RuntimeError without the PSPNet patch.
"""
import math
import os
import subprocess
import sys
import textwrap
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import determinism_ref as dr
import grad_ref as gr
from helpers import SA_LEVELS
from pvn3d_b200 import _ext, _lib, deterministic, synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, N = 24, 12288
SA_C = (6, 96, 256, 512)
FP_C = (256, 512, 512, 1024)


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


def _randn(shape, dev, seed):
    return torch.randn(shape, generator=torch.Generator(device=dev).manual_seed(seed), device=dev)


def _grads(op, g, idx, n, w=None):
    """(ordered, atomic, float32 restatement, float64 reference of grad_ref)"""
    with torch.inference_mode():
        fn = {"gather": _ext.gather_points_grad, "group": _ext.group_points_grad}.get(op)
        args = (g, idx, n) if w is None else (g, idx, w, n)
        fn = fn or _ext.three_interpolate_grad
        atomic = fn(*args)
        torch.use_deterministic_algorithms(True)
        try:
            ordered = fn(*args)
        finally:
            torch.use_deterministic_algorithms(False)
    if op == "gather":
        return ordered, atomic, dr.gather_grad32(g, idx, n), gr.gather_grad(g, idx, n)
    if op == "group":
        return ordered, atomic, dr.group_grad32(g, idx, n), gr.group_grad(g, idx, n)
    return ordered, atomic, dr.interp_grad32(g, idx, w, n), gr.interp_grad(g, idx, w, n)


def _check_all(op, g, idx, n, what, w=None):
    ordered, atomic, want, r64 = _grads(op, g, idx, n, w)
    dr.check_bits(ordered, want, what)
    gr.check(ordered, r64, what)
    gr.check_pair(ordered, atomic, r64, what + ": ordered vs atomic")
    return ordered


# ---- PointNet++ grads at the training shapes ------------------------------------------------------------------------
@pytest.mark.parametrize("ns_i", [0, 1])
@pytest.mark.parametrize("li", [0, 1, 2, 3])
def test_group_grad_ordered_training_shapes(cuda_dev, plan, li, ns_i):
    n, m, _, nss = SA_LEVELS[li]
    g = _randn((B, SA_C[li], m, nss[ns_i]), cuda_dev, 100 + 10 * li + ns_i)
    _check_all("group", g, plan.balls[(li, nss[ns_i])], n, f"group SA{li + 1} ns{nss[ns_i]}")


@pytest.mark.parametrize("lu", [0, 1, 2, 3])
def test_interp_grad_ordered_training_shapes(cuda_dev, plan, lu):
    idx, w = plan.nn[lu]
    n, m = plan.levels[lu].size(1), plan.levels[lu + 1].size(1)
    g = _randn((B, FP_C[lu], n), cuda_dev, 210 + lu)
    _check_all("interp", g, idx, m, f"interp FP{lu + 1}", w)


@pytest.mark.parametrize("li,c", [(0, 3), (1, 3), (2, 3), (3, 3), (1, 256)])
def test_gather_grad_ordered_training_shapes(cuda_dev, plan, li, c):
    n, m = SA_LEVELS[li][:2]
    _check_all("gather", _randn((B, c, m), cuda_dev, 300 + li + c), plan.fps[li], n, f"gather SA{li + 1} C{c}")


# ---- edges ----------------------------------------------------------------------------------------------------------
def test_group_grad_ordered_with_empty_balls(cuda_dev, plan):
    n, m, radii, nss = SA_LEVELS[1]
    centres = plan.levels[2].clone()
    centres[:, ::3] += 100.0
    idx = _ext.ball_query(centres, plan.levels[1], radii[1], nss[1])
    assert bool((idx[:, ::3] == 0).all())
    _check_all("group", _randn((B, SA_C[1], m, nss[1]), cuda_dev, 500), idx, n, "group, every third ball empty")


@pytest.mark.parametrize("m", [1, 2])
def test_interp_grad_ordered_over_one_or_two_known_points(cuda_dev, plan, m):
    unknown = plan.levels[2][:4]
    d2, idx = _ext.three_nn(unknown, plan.levels[3][:4, :m].contiguous())
    w = _weights(d2)
    _check_all("interp", _randn((4, 300, unknown.size(1)), cuda_dev, 601), idx, m, f"interp over {m} known", w)


def test_out_of_range_indices_contribute_nothing(cuda_dev, det_on):
    b, c, n, j = 3, 37, 500, 4096
    gen = torch.Generator(device=cuda_dev).manual_seed(700)
    idx = torch.randint(-50, n + 50, (b, j), generator=gen, device=cuda_dev, dtype=torch.int32)
    idx[0, :7] = torch.tensor([-2 ** 31, 2 ** 31 - 1, n, -1, n - 1, 0, n + 1], dtype=torch.int32)
    g = _randn((b, c, j), cuda_dev, 701)
    w = torch.rand((b, j, 3), generator=gen, device=cuda_dev)
    idx3 = torch.randint(-5, n + 5, (b, j, 3), generator=gen, device=cuda_dev, dtype=torch.int32)
    dr.check_bits(_ext.gather_points_grad(g, idx, n), dr.gather_grad32(g, idx, n), "gather, out-of-range")
    dr.check_bits(_ext.group_points_grad(g.reshape(b, c, j // 16, 16), idx.reshape(b, j // 16, 16), n),
                  dr.gather_grad32(g, idx, n), "group, out-of-range")
    dr.check_bits(_ext.three_interpolate_grad(g, idx3, w, n), dr.interp_grad32(g, idx3, w, n), "interp, out-of-range")


def _need(dev, nbytes):
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info(dev)
    if free < nbytes:
        pytest.skip(f"needs {nbytes / 2 ** 30:.1f} GiB of device memory, {free / 2 ** 30:.1f} free")


def test_ordered_gather_grad_reads_past_2_31(cuda_dev, det_on):
    c, m, n = 2048, 2 ** 20 + 3, 1024
    _need(cuda_dev, c * m * 4 + (2 << 30))
    try:
        v = (torch.arange(c, device=cuda_dev) % 7 + 1).float()
        g = v[None, :, None].expand(1, c, m).contiguous()
        idx = torch.randint(0, n, (1, m), generator=torch.Generator(device=cuda_dev).manual_seed(702),
                            device=cuda_dev, dtype=torch.int32)
        out = _ext.gather_points_grad(g, idx, n)
        want = v[:, None] * torch.bincount(idx[0].long(), minlength=n).float()[None]
        assert torch.equal(out[0], want), int((out[0] != want).sum())
    finally:
        g = idx = out = None
        torch.cuda.empty_cache()


def test_ordered_group_grad_writes_past_2_31(cuda_dev, det_on):
    c, n, npoints, ns = 1024, 2 ** 21 + 1, 64, 16
    _need(cuda_dev, c * n * 4 + (2 << 30))
    try:
        v = (torch.arange(c, device=cuda_dev) % 7 + 1).float()
        g = v[None, :, None, None].expand(1, c, npoints, ns).contiguous()
        lo = n - 300
        idx = torch.randint(lo, n, (1, npoints, ns), generator=torch.Generator(device=cuda_dev).manual_seed(703),
                            device=cuda_dev, dtype=torch.int32)
        idx[0, 0, 0] = n - 1
        out = _ext.group_points_grad(g, idx, n)
        want = v[:, None] * torch.bincount(idx.reshape(-1).long() - lo, minlength=n - lo).float()[None]
        assert torch.equal(out[0, :, lo:], want)
        for l0 in range(0, c, 64):
            assert not bool((out[0, l0:l0 + 64, :lo] != 0).any()), l0
    finally:
        g = idx = out = None
        torch.cuda.empty_cache()


def test_ordered_empty_shapes_and_batch_limit(cuda_dev):
    b, c, n = 3, 5, 40
    p = _lib.ptr
    st = torch.cuda.current_stream().cuda_stream
    lib = _lib.load()
    ef, ei, ew = (torch.empty((b, c, 0), device=cuda_dev), torch.empty((b, 0, 3), dtype=torch.int32, device=cuda_dev),
                  torch.empty((b, 0, 3), device=cuda_dev))
    for name, args in [("pvn3d_gather_points_grad_ordered", (p(ef), p(ei), b, c, n, 0)),
                       ("pvn3d_group_points_grad_ordered", (p(ef), p(ei), b, c, n, 0, 16)),
                       ("pvn3d_group_points_grad_ordered", (p(ef), p(ei), b, c, n, 7, 0)),
                       ("pvn3d_three_interpolate_grad_ordered", (p(ef), p(ei), p(ew), b, c, 0, n))]:
        out = torch.full((b, c, n), float("nan"), device=cuda_dev)
        assert getattr(lib, name)(*args, p(out), 0, 0, st) == 0, name
        assert torch.equal(out, torch.zeros_like(out)) and not bool(torch.signbit(out).any()), name
    bb = 65536
    g = torch.ones((bb, 1, 1), device=cuda_dev)
    i1 = torch.zeros((bb, 1, 1), dtype=torch.int32, device=cuda_dev)
    i3 = torch.zeros((bb, 1, 3), dtype=torch.int32, device=cuda_dev)
    w = torch.ones((bb, 1, 3), device=cuda_dev)
    assert lib.pvn3d_ordered_grad_workspace_bytes(bb, 1, 1) == 0
    for name, args in [("pvn3d_gather_points_grad_ordered", (p(g), p(i1), bb, 1, 1, 1)),
                       ("pvn3d_group_points_grad_ordered", (p(g), p(i1), bb, 1, 1, 1, 1)),
                       ("pvn3d_three_interpolate_grad_ordered", (p(g), p(i3), p(w), bb, 1, 1, 1))]:
        out = torch.full((bb, 1, 1), float("nan"), device=cuda_dev)
        rc = getattr(lib, name)(*args, p(out), 0, 0, st)
        torch.cuda.synchronize()
        assert rc == -2 and bool(torch.isnan(out).all()), (name, rc)
    # a short workspace is refused
    idx = torch.zeros((1, 8), dtype=torch.int32, device=cuda_dev)
    gg = torch.ones((1, 2, 8), device=cuda_dev)
    out = torch.empty((1, 2, 4), device=cuda_dev)
    need = lib.pvn3d_ordered_grad_workspace_bytes(1, 4, 8)
    ws = torch.empty(need - 1, dtype=torch.uint8, device=cuda_dev)
    assert lib.pvn3d_gather_points_grad_ordered(p(gg), p(idx), 1, 2, 4, 8, p(out), p(ws), need - 1, st) == -4


# ---- PSPNet pooling and upsampling ----------------------------------------------------------------------------------
def _pool_bwd(g, ih, iw):
    """the deterministic-mode backward of deterministic.adaptive_avg_pool2d: g [N,C,OH,OW]"""
    x = torch.zeros((g.size(0), g.size(1), ih, iw), device=g.device, requires_grad=True)
    deterministic.adaptive_avg_pool2d(x, tuple(g.shape[-2:])).backward(g)
    return x.grad


def _up_bwd(g, ih, iw, align, scale_factor=None):
    x = torch.zeros((g.size(0), g.size(1), ih, iw), device=g.device, requires_grad=True)
    size = None if scale_factor else tuple(g.shape[-2:])
    deterministic.interpolate(x, size=size, scale_factor=scale_factor, mode="bilinear", align_corners=align).backward(g)
    return x.grad


# the 1x1 prior is torch's mean (test_one_by_one_pool_is_torchs_own_op)
POOLS = [(60, 80, s, s) for s in (2, 3, 6)] + [(7, 7, 3, 3), (80, 80, 6, 6), (59, 59, 6, 6), (59, 80, 6, 7),
                                                  (5, 9, 8, 4)]
UPS = [(s, s, 60, 80, False, None) for s in (1, 2, 3, 6)] + [
    (60, 80, 120, 160, True, 2), (120, 160, 240, 320, True, 2), (240, 320, 480, 640, True, 2),
    (7, 5, 23, 17, False, None), (7, 5, 23, 17, True, None), (5, 3, 10, 6, False, 2.0), (13, 11, 4, 3, False, None)]


@pytest.mark.parametrize("case", POOLS, ids=[f"{a}x{b}->{c}x{d}" for a, b, c, d in POOLS])
def test_pool_backward(cuda_dev, det_on, case):
    ih, iw, oh, ow = case
    g = _randn((2, 3, oh, ow), cuda_dev, 800 + ih)
    got = _pool_bwd(g, ih, iw)
    want = dr.pool_backward32(g.reshape(6, oh, ow), ih, iw).reshape(got.shape)
    dr.check_bits(got, want, f"pool {case}")
    print(f"pool {case}: worst / bound {dr.check_bound(got.reshape(6, ih, iw), dr.pool_backward64(g.reshape(6, oh, ow), ih, iw)):.3g}")


@pytest.mark.parametrize("case", UPS, ids=[f"{a}x{b}->{c}x{d}-{e}-{f}" for a, b, c, d, e, f in UPS])
def test_upsample_backward(cuda_dev, det_on, case):
    ih, iw, oh, ow, align, sf = case
    g = _randn((2, 2, oh, ow), cuda_dev, 900 + ih)
    got = _up_bwd(g, ih, iw, align, sf)
    want = dr.upsample_backward32(g.reshape(4, oh, ow), ih, iw, align, sf).reshape(got.shape)
    dr.check_bits(got, want, f"upsample {case}")
    r = dr.upsample_backward64(g.reshape(4, oh, ow), ih, iw, align, sf)
    print(f"upsample {case}: worst / bound {dr.check_bound(got.reshape(4, ih, iw), r):.3g}")


SMALL_UPS = [c for c in UPS if c[0] * c[1] <= 64]     # one one-hot input per input element


@pytest.mark.parametrize("case", SMALL_UPS, ids=[f"{a}x{b}->{c}x{d}-{e}-{f}" for a, b, c, d, e, f in SMALL_UPS])
def test_upsample_taps_match_torch_forward(cuda_dev, case):
    """torch's forward of one-hot inputs is fl(lh lw) wherever one tap lands: pins the source indices and lambdas"""
    ih, iw, oh, ow, align, sf = case
    want = dr.upsample_forward_onehot(ih, iw, oh, ow, align, sf)
    for (y, x), w in want.items():
        e = torch.zeros((1, 1, ih, iw), device=cuda_dev)
        e[0, 0, y, x] = 1
        size = None if sf else (oh, ow)
        t = F.interpolate(e, size=size, scale_factor=sf, mode="bilinear", align_corners=align)[0, 0].cpu().numpy()
        ok = ~np.isnan(w)
        assert np.array_equal(t[ok].view(np.int32), w[ok].view(np.int32)), ((y, x), int((t[ok] != w[ok]).sum()))


@pytest.mark.parametrize("case", [(60, 80, 6, 8), (60, 80, 3, 4), (12, 16, 12, 16), (60, 80, 5, 8), (60, 80, 4, 8)])
def test_pool_backward_equals_torch_on_disjoint_bins(cuda_dev, case):
    """bins of 12 x 10 and 15 x 10 in the last two cases (a ratio that is not a power of two) and random gradients:
    (g / kH) / kW and (g / kW) / kH differ in about a third of the elements there, so this pins the order of the two
    divisions where bins are disjoint; the overlapping bins of test_single_contribution_equals_torch pin it there"""
    ih, iw, oh, ow = case
    g = _randn((2, 3, oh, ow), cuda_dev, 1000)
    x = torch.zeros((2, 3, ih, iw), device=cuda_dev, requires_grad=True)
    F.adaptive_avg_pool2d(x, (oh, ow)).backward(g)
    torch.use_deterministic_algorithms(True)
    try:
        got = _pool_bwd(g, ih, iw)
    finally:
        torch.use_deterministic_algorithms(False)
    dr.check_bits(got, x.grad, f"pool {case} vs torch")


def _one_hot_outputs(oh, ow):
    pts = {(0, 0), (oh - 1, ow - 1), (0, ow - 1), (oh - 1, 0), (oh // 2, ow // 3), (oh // 3 + 1, ow // 2 + 1)}
    return sorted(pts)


@pytest.mark.parametrize("kind", ["pool", "upsample"])
def test_single_contribution_equals_torch(cuda_dev, kind):
    """one nonzero output gradient: torch's atomic backward adds one term per input element (or the taps of one
    output in program order), so it is exact; the ordered kernel must give the same bits"""
    cases = ([(7, 7, 3, 3, None, None), (59, 80, 6, 6, None, None), (80, 80, 6, 6, None, None)] if kind == "pool"
             else [c for c in UPS if c[0] * c[1] <= 400])
    for ih, iw, oh, ow, align, sf in cases:
        for oy, ox in _one_hot_outputs(oh, ow):
            g = torch.zeros((1, 1, oh, ow), device=cuda_dev)
            g[0, 0, oy, ox] = float(_randn((1,), cuda_dev, 1050 + 97 * oy + ox))   # not a value both orders round alike
            x = torch.zeros((1, 1, ih, iw), device=cuda_dev, requires_grad=True)
            if kind == "pool":
                F.adaptive_avg_pool2d(x, (oh, ow)).backward(g)
            else:
                size = None if sf else (oh, ow)
                F.interpolate(x, size=size, scale_factor=sf, mode="bilinear", align_corners=align).backward(g)
            torch.use_deterministic_algorithms(True)
            try:
                got = _pool_bwd(g, ih, iw) if kind == "pool" else _up_bwd(g, ih, iw, align, sf)
            finally:
                torch.use_deterministic_algorithms(False)
            dr.check_bits(got, x.grad, f"{kind} {(ih, iw, oh, ow, align, sf)} output {(oy, ox)}")


def test_one_by_one_pool_is_torchs_own_op(cuda_dev, det_on):
    """a 1x1 output is torch's mean: same forward and backward bits as F.adaptive_avg_pool2d, no launch of ours, in
    either mode"""
    lib = _lib.load()
    x = _randn((2, 3, 60, 80), cuda_dev, 1120)
    for on in (True, False):
        torch.use_deterministic_algorithms(on)
        a, b = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        torch.cuda.synchronize()
        c0 = lib.pvn3d_launch_count()
        ya = deterministic.adaptive_avg_pool2d(a, (1, 1))
        ya.backward(torch.ones_like(ya))
        torch.cuda.synchronize()
        assert lib.pvn3d_launch_count() == c0
        yb = F.adaptive_avg_pool2d(b, (1, 1))
        yb.backward(torch.ones_like(yb))
        assert torch.equal(ya, yb) and torch.equal(a.grad, b.grad), on


def test_mode_off_runs_torch_backward(cuda_dev):
    """deterministic mode off: the wrapped ops give torch's forward bits and run torch's own (atomic) backward -- no
    launch of this library, and the same values up to the order of torch's atomics"""
    assert not torch.are_deterministic_algorithms_enabled()
    lib = _lib.load()
    cases = [(lambda x: deterministic.interpolate(x, size=(60, 80), mode="bilinear"),
              lambda x: F.interpolate(x, size=(60, 80), mode="bilinear"), (2, 3, 6, 6)),
             (lambda x: deterministic.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True),
              lambda x: F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True), (2, 3, 60, 80)),
             (lambda x: deterministic.adaptive_avg_pool2d(x, (6, 6)), lambda x: F.adaptive_avg_pool2d(x, (6, 6)),
              (2, 3, 59, 80))]
    for i, (mine, theirs, shape) in enumerate(cases):
        x = _randn(shape, cuda_dev, 1100 + i)
        a, b = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        ya, yb = mine(a), theirs(b)
        assert torch.equal(ya, yb), i
        g = _randn(ya.shape, cuda_dev, 1110 + i)
        torch.cuda.synchronize()
        c0 = lib.pvn3d_launch_count()
        ya.backward(g)
        torch.cuda.synchronize()
        assert lib.pvn3d_launch_count() == c0, i
        yb.backward(g)
        torch.testing.assert_close(a.grad, b.grad, rtol=1e-5, atol=1e-5 * float(g.abs().max()))


# ---- determinism itself ---------------------------------------------------------------------------------------------
def _step(plan, dev):
    """every ordered op once: group SA2, interp FP2, gather SA2, pool 60x80 -> 6, upsample 6 -> 60x80"""
    n, m, _, nss = SA_LEVELS[1]
    gg = _randn((B, SA_C[1], m, nss[1]), dev, 1200)
    gi = _randn((B, 64, n), dev, 1201)
    gc = _randn((B, 64, m), dev, 1202)
    gp = _randn((B, 32, 6, 6), dev, 1203)
    gu = _randn((B, 32, 60, 80), dev, 1204)
    idx, w = plan.nn[1]
    return lambda: [_ext.group_points_grad(gg, plan.balls[(1, nss[1])], n),
                    _ext.three_interpolate_grad(gi, idx, w, plan.levels[2].size(1)),
                    _ext.gather_points_grad(gc, plan.fps[1], n),
                    _pool_bwd(gp, 60, 80), _up_bwd(gu, 6, 6, False)]


def test_two_calls_and_two_streams_give_the_same_bits(cuda_dev, plan, det_on):
    run = _step(plan, cuda_dev)
    first = run()
    second = run()
    side = torch.cuda.Stream(cuda_dev)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        third = run()
    fourth = run()                          # concurrently with the side stream's work
    torch.cuda.synchronize()
    for i, (a, b, c, d) in enumerate(zip(first, second, third, fourth)):
        for o in (b, c, d):
            assert torch.equal(a.view(torch.int32), o.view(torch.int32)), i


def test_backward_makes_no_host_sync(cuda_dev, plan, det_on):
    run = _step(plan, cuda_dev)
    run()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        run()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_mode_off_launches_only_the_atomic_entry_points(cuda_dev, plan):
    """deterministic mode off: each _ext grad is exactly one launch, as the atomic entry point called directly; on:
    the ordered path's 3 + 3 p (keys, p radix passes, run starts, sums)"""
    lib = _lib.load()
    n, m, _, nss = SA_LEVELS[1]
    g = _randn((B, 8, m, nss[1]), cuda_dev, 1300)
    idx = plan.balls[(1, nss[1])]
    out = torch.empty((B, 8, n), device=cuda_dev)

    def count(fn):
        torch.cuda.synchronize()
        c0 = lib.pvn3d_launch_count()
        fn()
        return lib.pvn3d_launch_count() - c0

    direct = count(lambda: _lib.call("pvn3d_group_points_grad", cuda_dev, _lib.ptr(g), _lib.ptr(idx), B, 8, n, m,
                                     nss[1], _lib.ptr(out)))
    assert direct == 1
    assert count(lambda: _ext.group_points_grad(g, idx, n)) == direct
    assert count(lambda: _ext.gather_points_grad(g[:, :, :, 0].contiguous(), plan.fps[1], n)) == 1
    iw_idx, iw_w = plan.nn[1]
    gi = _randn((B, 8, n), cuda_dev, 1301)
    assert count(lambda: _ext.three_interpolate_grad(gi, iw_idx, iw_w, m)) == 1
    torch.use_deterministic_algorithms(True)
    try:
        passes = -(-(B * n).bit_length() // 8)        # 8-bit radix passes over the keys up to B * n
        assert count(lambda: _ext.group_points_grad(g, idx, n)) == 3 + 3 * passes
    finally:
        torch.use_deterministic_algorithms(False)


# ---- one training step of the staged reference PVN3D ----------------------------------------------------------------
STEP = textwrap.dedent("""
    import hashlib, json, sys
    import torch
    sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
    from helpers import load_reference_python
    from pvn3d_b200 import compat
    patch = sys.argv[1] == "patch"
    ref = load_reference_python()
    assert ref is not None
    if patch:
        compat.install(patch_deterministic=True)
    import lib.pvn3d as P
    from lib.loss import FocalLoss, OFLoss
    from lib.pspnet import Modified_PSPNet
    P.modified_psp_models["resnet34"] = lambda: Modified_PSPNet(sizes=(1, 2, 3, 6), psp_size=512,
                                                                deep_features_size=256, backend="resnet34",
                                                                pretrained=False)
    torch.use_deterministic_algorithms(True)
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    model = P.PVN3D(num_classes=22, pcld_input_channels=6, pcld_use_xyz=True, num_kps=8, num_points=12288).to(dev)
    model.train()
    crit, crit_of = FocalLoss(gamma=2), OFLoss()
    b, n = 2, 12288
    gen = torch.Generator().manual_seed(1)
    rgb = torch.rand((b, 3, 480, 640), generator=gen).to(dev)
    cld = torch.randn((b, n, 9), generator=gen).to(dev) * 0.1
    choose = torch.stack([torch.randperm(480 * 640, generator=gen)[:n] for _ in range(b)])[:, None].to(dev)
    labels = torch.randint(0, 22, (b, n), generator=gen).to(dev)
    kp_targ = torch.randn((b, n, 8, 3), generator=gen).to(dev) * 0.05
    ctr_targ = torch.randn((b, n, 1, 3), generator=gen).to(dev) * 0.05

    def run():
        torch.manual_seed(2)
        model.zero_grad(set_to_none=True)
        pred_kp_of, pred_rgbd_seg, pred_ctr_of = model(cld, rgb, choose)
        loss = (crit(pred_rgbd_seg.view(labels.numel(), -1), labels.view(-1)).sum() * 2.0
                + crit_of(pred_kp_of, kp_targ, labels).sum() + crit_of(pred_ctr_of, ctr_targ, labels).sum())
        loss.backward()
        torch.cuda.synchronize()
        return loss.detach().clone(), {{k: p.grad.detach().clone() for k, p in model.named_parameters()
                                        if p.grad is not None}}

    try:
        l1, g1 = run()
    except RuntimeError as e:
        print(json.dumps({{"raised": str(e)[:400]}}))
        sys.exit(0)
    l2, g2 = run()
    same = [k for k in g1 if torch.equal(g1[k].view(torch.int32), g2[k].view(torch.int32))]
    print(json.dumps({{"loss": [float(l1), float(l2)], "params": len(g1), "bit_equal": len(same),
                      "differ": [k for k in g1 if k not in same][:10]}}))
""")


def _run_step(mode):
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    code = STEP.format(root=ROOT, tests=os.path.join(ROOT, "tests"))
    r = subprocess.run([sys.executable, "-c", code, mode], capture_output=True, text=True, env=env, cwd=ROOT,
                       timeout=1200)
    assert r.returncode == 0, r.stderr[-3000:]
    import json
    return json.loads(r.stdout.strip().splitlines()[-1])


def _reference_staged():
    return os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "py", "lib"))


def test_pvn3d_training_step_repeats_bit_for_bit(cuda_dev):
    if not _reference_staged():
        pytest.skip("the reference Python is not staged under oracle/_ref/py")
    res = _run_step("patch")
    print(res)
    assert "raised" not in res, res
    assert res["loss"][0] == res["loss"][1] and math.isfinite(res["loss"][0])
    assert res["params"] > 100 and res["bit_equal"] == res["params"], res


def test_pvn3d_training_step_raises_without_the_pspnet_patch(cuda_dev):
    if not _reference_staged():
        pytest.skip("the reference Python is not staged under oracle/_ref/py")
    res = _run_step("plain")
    print(res)
    assert "raised" in res and "deterministic" in res["raised"], res
    assert "adaptive_avg_pool2d" in res["raised"] or "upsample_bilinear2d" in res["raised"], res
