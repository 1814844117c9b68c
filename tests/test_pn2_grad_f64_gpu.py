"""The three PointNet++ gradient ops (pvn3d_gather_points_grad, pvn3d_group_points_grad, pvn3d_three_interpolate_grad)
against float64 scatter references with the element-wise bound of tests/grad_ref.py, and the network's parameter
gradients through them.

  * training shapes: 24 frames x 12288 points (the reference's mini_batch_size), level clouds from the device's
    bit-exact FPS, ball-query / three_nn indices from `_ext` -- group at SA1-SA4 (nsample 16 and 32), interpolate at
    FP1-FP4 with the module's inverse-distance weights, gather at the four centre gathers and at 256 channels.  Every
    case runs with random-normal g (within the bound) and with integer g / dyadic weights (bit-equal);
  * contention and dispatch edges: every index 0 or n-1, empty balls, three_nn over 1 and 2 known points, c = 1, c not
    a multiple of the channel slices, c far above them, b = 1, a ragged last 256-slot block;
  * empty shapes (exact zeros over NaN-filled outputs), b = 65536 (refused, output untouched), outputs and inputs past
    2^31 elements;
  * the forward on a side stream with the backward through autograd;
  * every mutant of grad_ref rejected on a GPU case;
  * Pointnet2MSG in train() mode at 4 x 12288: the parameter gradients of the drop-in against a pure-torch fp32 twin
    and a float64 twin that replay the same FPS / ball-query / three_nn choices.
"""
import copy
import math
import types

import numpy as np
import pytest
import torch

import grad_ref as gr
from helpers import SA_LEVELS, load_reference_python
from pvn3d_b200 import _ext, _lib, pointnet2, synth, testing

pytestmark = pytest.mark.gpu

B, N = 24, 12288
SA_C = (6, 96, 256, 512)                            # feature channels grouped at SA1..SA4
FP_C = (256, 512, 512, 1024)                        # known-feature channels interpolated at FP1..FP4
KINDS = ("normal", "integer")


@pytest.fixture(autouse=True)
def _fp32_reference():
    """the module graphs below run in fp32 / float64, never TF32"""
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _weights(d2):
    """PointnetFPModule.forward's inverse-distance weights from squared distances (inf -> weight 0)"""
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
    nn = {}
    for lu in range(4):
        d2, idx = _ext.three_nn(levels[lu], levels[lu + 1])
        nn[lu] = (idx, _weights(d2))
    return types.SimpleNamespace(levels=levels, fps=fps, balls=balls, nn=nn)


def _g(shape, kind, dev, seed):
    gen = torch.Generator(device=dev).manual_seed(seed)
    if kind == "normal":
        return torch.randn(shape, generator=gen, device=dev)
    return torch.randint(-8, 9, shape, generator=gen, device=dev).float()


def _dyadic(shape, dev, seed):
    gen = torch.Generator(device=dev).manual_seed(seed)
    return torch.randint(0, 9, shape, generator=gen, device=dev).float() / 8


def _exact_ok(r, denom=1):
    """integer / dyadic terms: every partial sum is a multiple of 1/denom below 2^24 / denom -> exact in float32"""
    assert float(r.s.max()) * denom < 2 ** 24


def _check_group(g, idx, n, kind, what):
    got = _ext.group_points_grad(g, idx, n)
    r = gr.group_grad(g, idx, n)
    if kind == "integer":
        _exact_ok(r)
    gr.check(got, r, what, exact=kind == "integer")
    return got, r


def _check_gather(g, idx, n, kind, what):
    got = _ext.gather_points_grad(g, idx, n)
    r = gr.gather_grad(g, idx, n)
    if kind == "integer":
        _exact_ok(r)
    gr.check(got, r, what, exact=kind == "integer")
    return got, r


def _check_interp(g, idx, w, m, kind, what):
    got = _ext.three_interpolate_grad(g, idx, w, m)
    r = gr.interp_grad(g, idx, w, m)
    if kind == "integer":
        _exact_ok(r, 8)
    gr.check(got, r, what, exact=kind == "integer")
    return got, r


# ---- training shapes ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("ns_i", [0, 1])
@pytest.mark.parametrize("li", [0, 1, 2, 3])
def test_group_points_grad_training_shapes(cuda_dev, plan, li, ns_i, kind):
    n, m, _, nss = SA_LEVELS[li]
    ns = nss[ns_i]
    g = _g((B, SA_C[li], m, ns), kind, cuda_dev, 100 + 10 * li + ns_i)
    _check_group(g, plan.balls[(li, ns)], n, kind, f"group SA{li + 1} {n}->{m} C{SA_C[li]} ns{ns} {kind}")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("lu", [0, 1, 2, 3])
def test_three_interpolate_grad_training_shapes(cuda_dev, plan, lu, kind):
    idx, w = plan.nn[lu]
    n, m = plan.levels[lu].size(1), plan.levels[lu + 1].size(1)
    if kind == "integer":
        w = _dyadic(w.shape, cuda_dev, 200 + lu)
    g = _g((B, FP_C[lu], n), kind, cuda_dev, 210 + lu)
    _check_interp(g, idx, w, m, kind, f"interp FP{lu + 1} {n}<-{m} C{FP_C[lu]} {kind}")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("li,c", [(0, 3), (1, 3), (2, 3), (3, 3), (1, 256)])
def test_gather_points_grad_training_shapes(cuda_dev, plan, li, c, kind):
    n, m = SA_LEVELS[li][:2]
    g = _g((B, c, m), kind, cuda_dev, 300 + li + c)
    _check_gather(g, plan.fps[li], n, kind, f"gather SA{li + 1} {n}->{m} C{c} {kind}")


# ---- contention and dispatch edges ----------------------------------------------------------------------------------
def _sm_count(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


# name, b, c, n (points scattered into), j (slots = npoints * nsample, also the unknown count of interpolate), rule.
# c = None: chosen from the device's channel slices so that c is not a multiple of them and exceeds them
EDGES = [
    ("all index 0", 2, 37, 1000, 512 * 32, "zero"),
    ("all index n-1", 2, 37, 1000, 512 * 32, "last"),
    ("c = 1", 3, 1, 2000, 700 * 16, "random"),
    ("c not a multiple of the slices", 2, None, 3000, 2051, "random"),
    ("c >> slices, b = 1, one block", 1, 2000, 500, 200, "random"),
    ("one slice, every CTA loops all channels", 4, 64, 40000, 132 * 256, "random"),
    ("b = 1, ragged last block", 1, 19, 3000, 8 * 256 + 3, "random"),
]


def _edge_idx(rule, shape, n, dev, seed):
    if rule == "zero":
        return torch.zeros(shape, dtype=torch.int32, device=dev)
    if rule == "last":
        return torch.full(shape, n - 1, dtype=torch.int32, device=dev)
    gen = torch.Generator(device=dev).manual_seed(seed)
    return torch.randint(0, n, shape, generator=gen, device=dev, dtype=torch.int32)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", EDGES, ids=[e[0] for e in EDGES])
def test_grad_edges(cuda_dev, case, kind):
    name, b, c, n, j, rule = case
    slices = gr.channel_slices(1 << 30, b * math.ceil(j / 256), _sm_count(cuda_dev))
    if c is None:
        c = slices + slices // 2 + 1
        assert c % slices and c > slices, (c, slices)
    ns = 16 if j % 16 == 0 else 1
    idx = _edge_idx(rule, (b, j // ns, ns), n, cuda_dev, 400)
    print(f"[{name}] b {b} c {c} n {n} slots {j}: {min(slices, c)} channel slices")
    _check_group(_g((b, c, j // ns, ns), kind, cuda_dev, 401), idx, n, kind, f"group [{name}] {kind}")
    _check_gather(_g((b, c, j), kind, cuda_dev, 402), idx.reshape(b, j), n, kind, f"gather [{name}] {kind}")
    nn_idx = _edge_idx(rule, (b, j, 3), n, cuda_dev, 403)
    if kind == "integer":
        w = _dyadic((b, j, 3), cuda_dev, 404)
    else:
        w = torch.rand((b, j, 3), generator=torch.Generator(device=cuda_dev).manual_seed(404), device=cuda_dev)
        w = (w / w.sum(-1, keepdim=True)).contiguous()
    _check_interp(_g((b, c, j), kind, cuda_dev, 405), nn_idx, w, n, kind, f"interp [{name}] {kind}")


@pytest.mark.parametrize("kind", KINDS)
def test_group_grad_with_empty_balls(cuda_dev, plan, kind):
    """centres far from the cloud get all-zero index rows: index 0 of every frame takes nsample contributions each"""
    n, m, radii, nss = SA_LEVELS[1]
    xyz, centres = plan.levels[1], plan.levels[2].clone()
    centres[:, ::3] += 100.0
    idx = _ext.ball_query(centres, xyz, radii[1], nss[1])
    assert bool((idx[:, ::3] == 0).all())
    g = _g((B, SA_C[1], m, nss[1]), kind, cuda_dev, 500)
    _, r = _check_group(g, idx, n, kind, f"group SA2, every third ball empty, {kind}")
    assert int(r.k[:, 0, 0].min()) >= nss[1] * (m // 3)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("m", [1, 2])
def test_interp_grad_over_one_or_two_known_points(cuda_dev, plan, m, kind):
    """three_nn over m < 3 known points pads with index 0 at weight 0 (d2 = inf)"""
    unknown = plan.levels[2][:4]
    d2, idx = _ext.three_nn(unknown, plan.levels[3][:4, :m].contiguous())
    w = _weights(d2)
    assert bool((w[..., m:] == 0).all()) and bool((idx[..., m:] == 0).all())
    if kind == "integer":
        w = w.clone()
        w[..., :m] = _dyadic((4, unknown.size(1), m), cuda_dev, 600)
    g = _g((4, 300, unknown.size(1)), kind, cuda_dev, 601)
    _check_interp(g, idx, w, m, kind, f"interp over {m} known point(s) {kind}")


# ---- empty shapes and the batch limit -------------------------------------------------------------------------------
def _raw(name, *args):
    """the C entry point's return code (no raise), on the current stream"""
    return getattr(_lib.load(), name)(*args, torch.cuda.current_stream().cuda_stream)


def test_empty_shapes_write_zeros(cuda_dev):
    b, c, n = 3, 5, 40
    nan = float("nan")
    empty_f = torch.empty((b, c, 0), device=cuda_dev)
    empty_i = torch.empty((b, 0, 3), dtype=torch.int32, device=cuda_dev)
    empty_w = torch.empty((b, 0, 3), device=cuda_dev)
    zeros = torch.zeros((b, c, n), device=cuda_dev)
    for name, args in [
        ("pvn3d_gather_points_grad (m = 0)", ("pvn3d_gather_points_grad", empty_f, empty_i, b, c, n, 0)),
        ("pvn3d_group_points_grad (npoints = 0)", ("pvn3d_group_points_grad", empty_f, empty_i, b, c, n, 0, 16)),
        ("pvn3d_group_points_grad (nsample = 0)", ("pvn3d_group_points_grad", empty_f, empty_i, b, c, n, 7, 0)),
        ("pvn3d_three_interpolate_grad (n = 0)", ("pvn3d_three_interpolate_grad", empty_f, empty_i, empty_w, b, c, 0, n)),
    ]:
        out = torch.full((b, c, n), nan, device=cuda_dev)
        fn, *rest = args
        rest = [_lib.ptr(a) if isinstance(a, torch.Tensor) else a for a in rest]
        _lib.call(fn, cuda_dev, *rest, _lib.ptr(out))
        assert torch.equal(out, zeros) and not bool(torch.signbit(out).any()), name
    # the same through the drop-in's allocation
    assert torch.equal(_ext.gather_points_grad(torch.empty((b, c, 0), device=cuda_dev),
                                               torch.empty((b, 0), dtype=torch.int32, device=cuda_dev), n), zeros)
    assert torch.equal(_ext.group_points_grad(torch.empty((b, c, 0, 16), device=cuda_dev),
                                              torch.empty((b, 0, 16), dtype=torch.int32, device=cuda_dev), n), zeros)
    assert torch.equal(_ext.three_interpolate_grad(empty_f, empty_i, empty_w, n), zeros)


def test_batch_limit_refused_before_any_write(cuda_dev):
    b = 65536
    g = torch.ones((b, 1, 1), device=cuda_dev)
    idx = torch.zeros((b, 1, 1), dtype=torch.int32, device=cuda_dev)
    w = torch.ones((b, 1, 3), device=cuda_dev)
    idx3 = torch.zeros((b, 1, 3), dtype=torch.int32, device=cuda_dev)
    p = _lib.ptr
    for name, args in [("pvn3d_gather_points_grad", (p(g), p(idx), b, 1, 1, 1)),
                       ("pvn3d_group_points_grad", (p(g), p(idx), b, 1, 1, 1, 1)),
                       ("pvn3d_three_interpolate_grad", (p(g), p(idx3), p(w), b, 1, 1, 1))]:
        out = torch.full((b, 1, 1), float("nan"), device=cuda_dev)
        rc = _raw(name, *args, p(out))
        torch.cuda.synchronize()
        assert rc == -2, (name, rc)                  # PVN3D_ERR_UNSUPPORTED
        assert bool(torch.isnan(out).all()), name


# ---- past 2^31 elements ---------------------------------------------------------------------------------------------
def _need(dev, nbytes):
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info(dev)
    if free < nbytes:
        pytest.skip(f"needs {nbytes / 2 ** 30:.1f} GiB of device memory, {free / 2 ** 30:.1f} of "
                    f"{total / 2 ** 30:.1f} GiB free")


def _channel_values(c, dev):
    """small integers that differ between neighbouring channels: a wrong row stride reads or writes other values"""
    return (torch.arange(c, device=dev) % 7 + 1).float()


def test_gather_grad_reads_past_2_31(cuda_dev):
    c, m, n = 2048, 2 ** 20 + 3, 1024
    assert c * m > 2 ** 31
    _need(cuda_dev, c * m * 4 + (1 << 30))
    try:
        v = _channel_values(c, cuda_dev)
        g = v[None, :, None].expand(1, c, m).contiguous()
        gen = torch.Generator(device=cuda_dev).manual_seed(700)
        idx = torch.randint(0, n, (1, m), generator=gen, device=cuda_dev, dtype=torch.int32)
        out = torch.full((1, c, n), float("nan"), device=cuda_dev)
        _lib.call("pvn3d_gather_points_grad", cuda_dev, _lib.ptr(g), _lib.ptr(idx), 1, c, n, m, _lib.ptr(out))
        want = v[:, None] * torch.bincount(idx[0].long(), minlength=n).float()[None]
        assert torch.equal(out[0], want), int((out[0] != want).sum())
    finally:
        g = idx = out = None
        torch.cuda.empty_cache()


def test_group_grad_writes_past_2_31(cuda_dev):
    c, n, npoints, ns = 1024, 2 ** 21 + 1, 64, 16
    assert c * n > 2 ** 31
    _need(cuda_dev, c * n * 4 + (1 << 30))
    try:
        v = _channel_values(c, cuda_dev)
        g = v[None, :, None, None].expand(1, c, npoints, ns).contiguous()
        lo = n - 300
        gen = torch.Generator(device=cuda_dev).manual_seed(701)
        idx = torch.randint(lo, n, (1, npoints, ns), generator=gen, device=cuda_dev, dtype=torch.int32)
        idx[0, 0, 0] = n - 1
        out = torch.full((1, c, n), float("nan"), device=cuda_dev)
        _lib.call("pvn3d_group_points_grad", cuda_dev, _lib.ptr(g), _lib.ptr(idx), 1, c, n, npoints, ns, _lib.ptr(out))
        want = v[:, None] * torch.bincount(idx.reshape(-1).long() - lo, minlength=n - lo).float()[None]
        assert torch.equal(out[0, :, lo:], want), int((out[0, :, lo:] != want).sum())
        for l0 in range(0, c, 64):                   # the memset reached every row, past 2^31 included
            assert not bool((out[0, l0:l0 + 64, :lo] != 0).any()), l0
    finally:
        g = idx = out = None
        torch.cuda.empty_cache()


# ---- streams --------------------------------------------------------------------------------------------------------
def test_autograd_backward_of_a_side_stream_forward(cuda_dev, plan):
    """forward on a side stream, backward through autograd (which runs each backward on its forward's stream): within
    the bound of float64 and of the default-stream result, and two runs agree within the bound"""
    n, m, _, nss = SA_LEVELS[1]
    feats = torch.randn((B, SA_C[1], n), device=cuda_dev)
    centres_idx = plan.fps[1]
    ball = plan.balls[(1, nss[1])]
    nn_idx, nn_w = plan.nn[1]
    known = torch.randn((B, FP_C[1], m), device=cuda_dev)
    rg = torch.randn((B, SA_C[1], m, nss[1]), device=cuda_dev)
    rc = torch.randn((B, SA_C[1], m), device=cuda_dev)
    ri = torch.randn((B, FP_C[1], n), device=cuda_dev)
    refs = {"group": gr.group_grad(rg, ball, n), "gather": gr.gather_grad(rc, centres_idx, n),
            "interp": gr.interp_grad(ri, nn_idx, nn_w, m)}

    def run(stream):
        f = feats.clone().requires_grad_(True)
        k = known.clone().requires_grad_(True)
        stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):
            loss = ((pointnet2.grouping_operation(f, ball) * rg).sum()
                    + (pointnet2.gather_operation(f, centres_idx) * rc).sum())
            loss_i = (pointnet2.three_interpolate(k, nn_idx, nn_w) * ri).sum()
        loss.backward()
        loss_i.backward()
        torch.cuda.synchronize()
        return f.grad, k.grad

    side = torch.cuda.Stream(cuda_dev)
    runs = [run(side), run(torch.cuda.current_stream()), run(side)]
    wants = {"feats": gr.Ref(refs["group"].ref + refs["gather"].ref, refs["group"].k + refs["gather"].k,
                             refs["group"].s + refs["gather"].s), "known": refs["interp"]}
    for i, (what, r) in enumerate(wants.items()):
        for name, got in zip(("side", "default", "side again"), (x[i] for x in runs)):
            gr.check(got, r, f"{what} grad, {name} stream")
        gr.check_pair(runs[0][i], runs[1][i], r, f"{what}: side vs default stream")
        gr.check_pair(runs[0][i], runs[2][i], r, f"{what}: two side-stream runs")


# ---- mutants --------------------------------------------------------------------------------------------------------
MUTANTS = ["dedup", "frame0", "shift", "last channel", "last slice", "swapped weights", "drop one", "drop one interp",
           "reference wrapper"]


@pytest.mark.parametrize("mutant", MUTANTS)
def test_mutants_rejected_on_gpu_cases(cuda_dev, plan, mutant):
    if mutant in ("swapped weights", "drop one interp", "reference wrapper"):
        idx, w = plan.nn[1]
        n, m = plan.levels[1].size(1), plan.levels[2].size(1)
        g = _g((B, FP_C[1], n), "normal", cuda_dev, 800)
        _, r = _check_interp(g, idx, w, m, "normal", "interp FP2")
        if mutant == "swapped weights":
            bad = gr.interp_grad(g, idx, gr.mut_swap_nn_weights(w), m).ref.float()
        elif mutant == "drop one interp":
            bad = gr.mut_drop_one(gr.interp_terms(g, w), idx.reshape(B, -1), r)
        else:
            bad = torch.from_numpy(gr.mut_reference_wrapper(g.cpu().numpy(), idx.cpu().numpy(), w.cpu().numpy(), m))
            bad = bad.to(cuda_dev)
    elif mutant == "last slice":
        b, c, n, j = 1, 2000, 500, 200                # one 256-slot block: c / grid.y channels per slice
        slices = gr.channel_slices(c, 1, _sm_count(cuda_dev))
        assert 1 < slices < c
        idx = _edge_idx("random", (b, j, 1), n, cuda_dev, 801)
        g = _g((b, c, j, 1), "normal", cuda_dev, 802)
        _, r = _check_group(g, idx, n, "normal", "group, one block")
        bad = gr.mut_drop_channels(r, range(slices - 1, c, slices))
    else:
        n, m, _, nss = SA_LEVELS[1]
        idx = plan.balls[(1, nss[1])]
        g = _g((B, SA_C[1], m, nss[1]), "normal", cuda_dev, 803)
        _, r = _check_group(g, idx, n, "normal", "group SA2")
        bad = {"dedup": lambda: gr.mut_group_dedup(g, idx, n),
               "frame0": lambda: gr.mut_frames(r, "frame0"),
               "shift": lambda: gr.mut_frames(r, "shift"),
               "last channel": lambda: gr.mut_drop_channels(r, [SA_C[1] - 1]),
               "drop one": lambda: gr.mut_drop_one(g.reshape(B, SA_C[1], -1), idx.reshape(B, -1), r)}[mutant]()
    with pytest.raises(AssertionError, match="outside the bound"):
        gr.check(bad, r, f"mutant {mutant}")


# ---- the network's parameter gradients ------------------------------------------------------------------------------
_DISCRETE = ("furthest_point_sample", "ball_query", "three_nn")


def _t_gather(features, idx):
    b, c = features.shape[:2]
    return features.gather(2, idx.long()[:, None].expand(b, c, idx.size(1)))


def _t_group(features, idx):
    b, c = features.shape[:2]
    return features.gather(2, idx.long().reshape(b, 1, -1).expand(b, c, -1)).reshape(b, c, *idx.shape[1:])


def _t_interp(features, idx, weight):
    return (_t_group(features, idx) * weight[:, None]).sum(-1)


def _recorder(log):
    orig = {k: getattr(pointnet2, k) for k in _DISCRETE}

    def wrap(name):
        def fn(*a):
            out = orig[name](*a)
            log[name].append(out)
            return out
        return fn
    return {k: wrap(k) for k in _DISCRETE}


def _twin(log, f64):
    its = {k: iter(v) for k, v in log.items()}

    def nn(unknown, known):
        dist, idx = next(its["three_nn"])
        if f64:                                          # the same neighbours, their float64 distances
            b, n = idx.shape[:2]
            k = known.detach().gather(1, idx.long().reshape(b, -1, 1).expand(b, n * 3, 3)).reshape(b, n, 3, 3)
            dist = (unknown.detach()[:, :, None] - k).square().sum(-1).sqrt()
        return dist, idx

    return {"furthest_point_sample": lambda xyz, npoint: next(its["furthest_point_sample"]),
            "ball_query": lambda radius, nsample, xyz, new_xyz: next(its["ball_query"]),
            "three_nn": nn, "gather_operation": _t_gather, "grouping_operation": _t_group,
            "three_interpolate": _t_interp}


def _arm(model, pc, r, ops, monkeypatch):
    with monkeypatch.context() as mp:
        for k, fn in ops.items():
            mp.setattr(pointnet2, k, fn)
        x = pc.detach().clone().requires_grad_(True)
        (model(x) * r).sum().backward()
    grads = {k: p.grad.detach().double() for k, p in model.named_parameters()}
    grads["input"] = x.grad.detach().double()
    return grads


def _err(g, g64):
    """(mean, 99.9th percentile) of |g - g64| / mean |g64|"""
    e = ((g - g64).abs() / g64.abs().mean()).flatten()
    return float(e.mean()), float(e.kthvalue(max(1, math.ceil(0.999 * e.numel()))).values)


def test_pointnet2msg_parameter_gradients_train_mode(cuda_dev, monkeypatch):
    b = 4
    frames = synth.make_batch("ycb", b, n_points=N, config_id=32)
    pc = torch.from_numpy(np.stack([f.cld_rgb_nrm for f in frames])).to(cuda_dev)
    model = testing.seeded_pointnet2msg(0, 1).to(cuda_dev).train()
    state = copy.deepcopy(model.state_dict())
    twin32 = copy.deepcopy(model)
    twin64 = copy.deepcopy(model).double()
    r = torch.randn((b, 128, N), generator=torch.Generator(device=cuda_dev).manual_seed(900), device=cuda_dev)

    log = {k: [] for k in _DISCRETE}
    arms = {"drop-in": _arm(model, pc, r, _recorder(log), monkeypatch)}
    assert [len(log[k]) for k in _DISCRETE] == [4, 8, 4]
    arms["torch fp32"] = _arm(twin32, pc, r, _twin(log, False), monkeypatch)
    g64 = _arm(twin64, pc.double(), r.double(), _twin(log, True), monkeypatch)

    ref = load_reference_python()
    if ref is not None:
        rmod = ref.pvn3d.Pointnet2MSG(input_channels=6)
        rmod.load_state_dict(state, strict=True)
        arms["reference module"] = _arm(rmod.to(cuda_dev).train(), pc, r, {}, monkeypatch)
        assert set(arms["reference module"]) == set(g64)
    else:
        print("reference Python not staged: the reference module's arm is skipped")

    base = "torch fp32"
    worst = {k: 0.0 for k in arms if k != base}
    for name in g64:
        if float(g64[name].abs().mean()) == 0.0:
            assert all(float(a[name].abs().max()) == 0.0 for a in arms.values()), name
            continue
        eb = _err(arms[base][name], g64[name])
        line = [f"{name}: {base} mean {eb[0]:.3g} p99.9 {eb[1]:.3g}"]
        for arm, grads in arms.items():
            if arm == base:
                continue
            ea = _err(grads[name], g64[name])
            line.append(f"{arm} mean {ea[0]:.3g} p99.9 {ea[1]:.3g}")
            assert ea[0] <= 2 * eb[0] + 1e-6 and ea[1] <= 2 * eb[1] + 1e-6, (arm, name, ea, eb)
            worst[arm] = max(worst[arm], (ea[0] - 1e-6) / (2 * eb[0]), (ea[1] - 1e-6) / (2 * eb[1]))
        print("; ".join(line))
    print("largest (error - 1e-6) / (2 x torch fp32 error) per arm:", {k: round(v, 3) for k, v in worst.items()})
