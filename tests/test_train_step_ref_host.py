"""tests/train_step_ref.py on CPU tensors at small shapes (no GPU): the replay ops of the training-step twin and their
autograd gradients against tests/grad_ref.py's float64 scatter adjoints, the 16-bit replay's single rounding, and the
error statistic and bound of tests/test_train_step_f64_gpu.py rejecting each of its mutants on synthetic gradients."""
import numpy as np
import pytest
import torch

import grad_ref as gr
import train_ref
import train_step_ref as R

B, C, N, M, S = 2, 5, 40, 9, 6


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _idx(shape, n, seed):
    return torch.randint(0, n, shape, generator=_gen(seed), dtype=torch.int32)


def _weights(shape, seed):
    w = torch.rand(shape, generator=_gen(seed), dtype=torch.float64) + 0.1
    return w / w.sum(-1, keepdim=True)


def _close(got, want):
    torch.testing.assert_close(got, want, rtol=1e-13, atol=1e-15)


# ---- the replay ops against the float64 adjoints ---------------------------------------------------------------------
def test_group_replay_and_gradient_equal_the_f64_adjoint():
    f = torch.randn((B, C, N), generator=_gen(1), dtype=torch.float64, requires_grad=True)
    idx = _idx((B, M, S), N, 2)
    out = R.Group.apply(f, idx)
    want = torch.stack([f[b][:, idx[b].long()] for b in range(B)])
    assert out.shape == (B, C, M, S) and torch.equal(out, want)
    g = torch.randn(out.shape, generator=_gen(3), dtype=torch.float64)
    out.backward(g)
    _close(f.grad, gr.group_grad(g, idx, N).ref)


def test_gather_replay_and_gradient_equal_the_f64_adjoint():
    f = torch.randn((B, 3, N), generator=_gen(4), dtype=torch.float64, requires_grad=True)
    idx = _idx((B, M), N, 5)
    out = R.Group.apply(f, idx)
    assert out.shape == (B, 3, M) and torch.equal(out, torch.stack([f[b][:, idx[b].long()] for b in range(B)]))
    g = torch.randn(out.shape, generator=_gen(6), dtype=torch.float64)
    out.backward(g)
    _close(f.grad, gr.gather_grad(g, idx, N).ref)


def test_interp_replay_and_gradient_equal_the_f64_adjoint():
    f = torch.randn((B, C, M), generator=_gen(7), dtype=torch.float64, requires_grad=True)
    idx, w = _idx((B, N, 3), M, 8), _weights((B, N, 3), 9)
    out = R.Interp.apply(f, idx, w)
    want = torch.stack([(f[b][:, idx[b].long()] * w[b][None]).sum(-1) for b in range(B)])
    _close(out, want)
    g = torch.randn(out.shape, generator=_gen(10), dtype=torch.float64)
    out.backward(g)
    _close(f.grad, gr.interp_grad(g, idx, w, M).ref)


def test_twin_replays_the_recorded_choices():
    xyz = torch.rand((B, N, 3), generator=_gen(11), dtype=torch.float64)
    known = xyz[:, :M].contiguous()
    nn_idx = _idx((B, N, 3), M, 12)
    log = {"furthest_point_sample": [_idx((B, M), N, 13)], "ball_query": [_idx((B, M, S), N, 14)],
           "three_nn": [(torch.rand((B, N, 3), dtype=torch.float32), nn_idx)]}
    ops = R.twin(log, f64=True)
    assert ops["furthest_point_sample"](xyz.float(), M) is log["furthest_point_sample"][0]
    assert ops["ball_query"](0.1, S, xyz.float(), known.float()) is log["ball_query"][0]
    dist, idx = ops["three_nn"](xyz, known)
    assert idx is nn_idx and dist.dtype == torch.float64
    want = np.linalg.norm(xyz.numpy()[:, :, None] - np.stack([known.numpy()[b][nn_idx[b].long().numpy()]
                                                              for b in range(B)]), axis=-1)
    np.testing.assert_allclose(dist.numpy(), want, rtol=1e-15)
    rec = R.twin({k: list(v) for k, v in log.items()}, f64=False)["three_nn"](xyz.float(), known.float())
    assert rec[0] is log["three_nn"][0][0] and rec[1] is nn_idx
    seen = {k: [] for k in R.DISCRETE}
    wrapped = R.recorder(seen, {k: (lambda *a, k=k: (k, len(a))) for k in R.DISCRETE})
    assert wrapped["ball_query"](0.1, S, xyz, known) == ("ball_query", 4) and seen["ball_query"] == [("ball_query", 4)]


# ---- the 16-bit contract ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_16_bit_replay_rounds_once(dt):
    f = (torch.randn((B, C, M), generator=_gen(20)) * 3).to(dt)
    idx, w = _idx((B, N, 3), M, 21), _weights((B, N, 3), 22).float()
    out = R.Interp.apply(f, idx, w)
    want = R.Interp.apply(f.float(), idx, w).to(dt)                     # the float32 op, rounded once
    assert out.dtype == dt and torch.equal(out.view(torch.int16), want.view(torch.int16))

    # 300 unit gradients land on point 0: float32 sums reach 300 (a 16-bit value); a sum kept in 16 bits sticks at
    # 256 in bfloat16, whose spacing there is 2, and the replay must not do that
    idx0 = torch.zeros((1, 50, 6), dtype=torch.int32)
    f0 = torch.zeros((1, 1, 4), dtype=dt, requires_grad=True)
    out0 = R.Group.apply(f0, idx0)
    out0.backward(torch.ones_like(out0))
    assert f0.grad.dtype == dt and float(f0.grad[0, 0, 0]) == 300.0 and float(f0.grad[0, 0, 1:].abs().max()) == 0
    if dt == torch.bfloat16:
        acc = torch.zeros((), dtype=dt)
        for _ in range(300):
            acc = acc + torch.ones((), dtype=dt)
        assert float(acc) == 256.0                                       # what rounding after every term gives

    # integer gradients and dyadic weights: the float32 sums are exact, so each replayed gradient is round16 of the
    # float64 adjoint, bit for bit
    g = torch.randint(-4, 5, (B, C, M, S), generator=_gen(23)).to(dt)
    gidx = _idx((B, M, S), N, 24)
    fs = torch.zeros((B, C, N), dtype=dt, requires_grad=True)
    R.Group.apply(fs, gidx).backward(g)
    assert torch.equal(fs.grad.view(torch.int16), gr.group_grad(g, gidx, N).ref.to(dt).view(torch.int16))
    gi = torch.randint(-8, 9, (B, C, N), generator=_gen(25)).to(dt)
    wd = torch.randint(0, 9, (B, N, 3), generator=_gen(26)).float() / 8
    fk = torch.zeros((B, C, M), dtype=dt, requires_grad=True)
    R.Interp.apply(fk, idx, wd).backward(gi)
    assert torch.equal(fk.grad.view(torch.int16), gr.interp_grad(gi, idx, wd, M).ref.to(dt).view(torch.int16))


# ---- the statistic, the bound and the mutants ------------------------------------------------------------------------
def _fp32_scatter(terms, idx, n, reverse=False):
    """a float32 scatter-add of terms [B,C,J] at idx [B,J], in slot order or its reverse"""
    b, c, j = terms.shape
    out = torch.zeros((b, c, n), dtype=torch.float32)
    order = torch.arange(j - 1, -1, -1) if reverse else torch.arange(j)
    for s in order.tolist():
        out[torch.arange(b)[:, None], torch.arange(c)[None], idx[:, s].long()[:, None]] += terms[:, :, s].float()
    return out


def _accepts(arm, twin, g64, floor=1e-6, scale=None):
    return R.within(R.err(arm, g64, scale), R.err(twin, g64, scale), floor)


def _group_case():
    g = torch.randn((B, 16, 64, 8), generator=_gen(30), dtype=torch.float64)
    idx = torch.randint(0, 48, (B, 64, 8), generator=_gen(31), dtype=torch.int32)
    flat_g, flat_i = g.reshape(B, 16, -1), idx.reshape(B, -1)
    return g, idx, gr.group_grad(g, idx, 48).ref, _fp32_scatter(flat_g, flat_i, 48), \
        _fp32_scatter(flat_g, flat_i, 48, reverse=True)


def test_first_of_run_marks_the_lowest_slot_of_each_point():
    idx = torch.tensor([[[3, 1], [3, 0]], [[2, 2], [0, 2]]], dtype=torch.int32)
    assert R.first_of_run(idx).tolist() == [[True, True, False, True], [True, False, True, False]]
    _, idx, *_ = _group_case()
    first = R.first_of_run(idx)
    flat = idx.reshape(B, -1).long()
    for b in range(B):
        marked = flat[b][first[b]]
        assert len(set(marked.tolist())) == len(marked) == len(set(flat[b].tolist()))


def test_fp32_orders_pass_and_the_dropped_slot_fails():
    g, idx, g64, twin, arm = _group_case()
    assert not torch.equal(twin, arm)                                   # the two orders differ in some bits
    assert _accepts(arm, twin, g64)
    bad = gr.group_grad(R.drop_first_of_run(g, idx), idx, 48).ref.float()
    assert not _accepts(bad, twin, g64)


def test_swapped_interpolation_weights_fail():
    g = torch.randn((B, 16, 96), generator=_gen(32), dtype=torch.float64)
    idx, w = _idx((B, 96, 3), 30, 33), _weights((B, 96, 3), 34)
    g64 = gr.interp_grad(g, idx, w, 30).ref
    terms = gr.interp_terms(g, w.float())
    twin = _fp32_scatter(terms, idx.reshape(B, -1), 30)
    arm = _fp32_scatter(terms, idx.reshape(B, -1), 30, reverse=True)
    assert _accepts(arm, twin, g64)
    bad = gr.interp_grad(g, idx, R.swap_pairs(w), 30).ref.float()
    assert not _accepts(bad, twin, g64)
    assert torch.equal(R.swap_pairs(R.swap_pairs(w)), w)
    odd = _weights((1, 5, 3), 35)
    assert torch.equal(R.swap_pairs(odd)[0, 4], odd[0, 4]) and torch.equal(R.swap_pairs(odd)[0, 0], odd[0, 1])


def test_flipped_align_corners_fails():
    go = torch.randn((2, 8, 32, 40), generator=_gen(36), dtype=torch.float64)

    def bw(g, align):
        return torch.ops.aten.upsample_bilinear2d_backward(g, [32, 40], [2, 8, 16, 20], align, 2.0, 2.0)
    g64 = bw(go, True)
    twin = bw(go.float(), True)
    assert _accepts(twin, twin, g64)
    assert not _accepts(bw(go.float(), False), twin, g64)


def test_scaled_loss_gradient_fails():
    _, _, g64, twin, arm = _group_case()
    assert _accepts(arm, twin, g64)
    assert not _accepts(arm * R.LOSS_SCALE_MUTANT, twin, g64)


def test_ratio_and_families():
    assert R.ratio((2.5e-6, 4e-6), (1e-6, 2e-6), 1e-6) == pytest.approx(0.75)
    assert R.within((2.5e-6, 4e-6), (1e-6, 2e-6), 1e-6) and not R.within((3.5e-6, 4e-6), (1e-6, 2e-6), 1e-6)
    assert [R.family(k) for k in ("cnn.model.up_1.conv.1.bias", "pointnet2.SA_modules.0.mlps.0.layer0.conv.weight",
                                  "rgbd_feat.conv3.weight", "KpOF_layer.0.conv.weight")] == \
        ["CNN", "PointNet++", "DenseFusion", "heads"]


def test_frames_are_two_real_scenes():
    depth, K, cs, rgb, label, ids, rts = train_ref.raw_frames(2)
    assert depth.shape == label.shape == (2, 480, 640) and rgb.shape == (2, 3, 480, 640)
    assert (depth > 0).all() and all((label[f] > 0).sum() > 1000 for f in range(2))
    assert ids[:, :4].tolist() == [[1, 4, 9, 4]] * 2 and np.allclose(rts[:, :4, :, :3] @ rts[:, :4, :, :3].transpose(
        0, 1, 3, 2), np.eye(3))
    sparse = train_ref.raw_frames(2, sparse=(1,))                      # the same draws, frame 1 with 300 valid pixels
    assert int((sparse[0][1] > 0).sum()) == 300 and np.array_equal(sparse[0][0], depth[0])
    assert all(np.array_equal(a, b) for a, b in zip(sparse[1:], (K, cs, rgb, label, ids, rts)))


def test_err_with_a_per_element_scale():
    g64 = torch.tensor([1e-17, -2e-17], dtype=torch.float64)
    g = torch.tensor([3e-9, -1e-9])
    sums = torch.tensor([1e-2, 1e-3], dtype=torch.float64)
    mean, p999 = R.err(g, g64, sums)
    want = (g.double() - g64).abs() / sums
    assert mean == pytest.approx(float(want.mean())) and p999 == pytest.approx(float(want.max()))
