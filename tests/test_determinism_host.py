"""The restatements of tests/determinism_ref.py against their float64 adjoints on small cases, and the mutants each
check must reject (no GPU)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import determinism_ref as dr


def _g(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


def _padded_balls(b, m, s, n, seed):
    """ball rows as ball query pads them: a random number of hits, the rest repeats of the first (all 0 when empty)"""
    rng = np.random.default_rng(seed)
    idx = np.zeros((b, m, s), np.int32)
    for f in range(b):
        for j in range(m):
            k = int(rng.integers(0, s + 1))
            hits = np.sort(rng.choice(n, size=k, replace=False)) if k else np.zeros(0, np.int32)
            idx[f, j, :k] = hits
            idx[f, j, k:] = hits[0] if k else 0
    return torch.from_numpy(idx)


def test_group_restatement_within_the_adjoint_bound():
    b, c, m, s, n = 2, 5, 40, 16, 100
    idx = _padded_balls(b, m, s, n, 0)
    g = _g((b, c, m, s), 1)
    r = dr.scatter64(g.reshape(b, c, -1), idx.reshape(b, -1), n)
    dr.check_bound(dr.group_grad32(g, idx, n), r, "group")
    assert int(r.k.max()) > s                       # padding piles many slots onto index 0


def test_every_slot_on_one_point():
    b, c, j, n = 1, 3, 500, 4
    idx = torch.zeros((b, j), dtype=torch.int32)
    g = _g((b, c, j), 2)
    got = dr.gather_grad32(g, idx, n)
    want = torch.zeros(c)
    for t in range(j):                              # the loop the contract spells
        want = want + g[0, :, t]
    dr.check_bits(got[0, :, 0], want, "one point, every slot")
    assert torch.equal(got[0, :, 1:], torch.zeros((c, n - 1))) and not bool(torch.signbit(got[0, :, 1:]).any())
    dr.check_bound(got, dr.scatter64(g, idx, n), "one point")


def test_interp_restatement_within_the_adjoint_bound():
    b, c, n, m = 2, 4, 300, 20
    gen = torch.Generator().manual_seed(3)
    idx = torch.randint(0, m, (b, n, 3), generator=gen, dtype=torch.int32)
    w = torch.rand((b, n, 3), generator=gen)
    w = w / w.sum(-1, keepdim=True)
    g = _g((b, c, n), 4)
    r = dr.scatter64(dr.interp_terms64(g, w), idx.reshape(b, -1), m)
    dr.check_bound(dr.interp_grad32(g, idx, w, m), r, "interp")


def test_out_of_range_entries_are_dropped():
    g = _g((1, 2, 6), 5)
    idx = torch.tensor([[0, -1, 3, 7, 3, 2 ** 31 - 1]], dtype=torch.int32)
    got = dr.gather_grad32(g, idx, 4)
    want = torch.zeros((1, 2, 4))
    want[0, :, 0] = g[0, :, 0]
    want[0, :, 3] = g[0, :, 2] + g[0, :, 4]
    dr.check_bits(got, want, "out of range")


@pytest.mark.parametrize("case", [(7, 7, 3, 3), (80, 80, 6, 6), (59, 59, 6, 6), (60, 80, 6, 6), (5, 9, 8, 4)])
def test_pool_restatement_within_the_adjoint_bound(case):
    ih, iw, oh, ow = case
    g = _g((3, oh, ow), 6)
    r = dr.pool_backward64(g, ih, iw)
    dr.check_bound(dr.pool_backward32(g, ih, iw), r, f"pool {case}")
    x = torch.zeros((1, 3, ih, iw), dtype=torch.float64, requires_grad=True)
    F.adaptive_avg_pool2d(x, (oh, ow)).backward(g.double()[None])
    assert torch.allclose(x.grad[0], r.ref, rtol=1e-12, atol=1e-15)   # the adjoint is torch's own in float64


@pytest.mark.parametrize("case", [(1, 1, 60, 80, False), (2, 2, 60, 80, False), (3, 3, 60, 80, False),
                                  (6, 6, 60, 80, False), (6, 8, 12, 16, True), (7, 5, 23, 17, False),
                                  (7, 5, 23, 17, True)])
def test_upsample_restatement_within_the_adjoint_bound(case):
    ih, iw, oh, ow, align = case
    g = _g((2, oh, ow), 7)
    r = dr.upsample_backward64(g, ih, iw, align)
    dr.check_bound(dr.upsample_backward32(g, ih, iw, align), r, f"upsample {case}")
    x = torch.zeros((1, 2, ih, iw), dtype=torch.float64, requires_grad=True)
    F.interpolate(x, size=(oh, ow), mode="bilinear", align_corners=align).backward(g.double()[None])
    # float32 lambdas against torch's float64 ones: a few float32 ulps of the source index per term
    assert float((x.grad[0] - r.ref).abs().max()) <= 1e-5 * float(r.s.max())


def test_upsample_taps_match_torch_forward_on_cpu_where_single():
    """torch's CPU forward of one-hot inputs, at the single-tap outputs of the PSPNet priors: the same lambdas"""
    for s in (1, 3, 6):
        for (y, x), w in dr.upsample_forward_onehot(s, s, 60, 80, False).items():
            e = torch.zeros((1, 1, s, s))
            e[0, 0, y, x] = 1
            t = F.interpolate(e, size=(60, 80), mode="bilinear", align_corners=False)[0, 0].numpy()
            ok = ~np.isnan(w)
            assert np.array_equal(t[ok], w[ok]), (s, y, x)


# ---- mutants --------------------------------------------------------------------------------------------------------
def test_reversed_order_is_rejected():
    g = dr.cancelling_terms(8, 64, 8)
    idx = torch.zeros((1, 64), dtype=torch.int32)
    idx[0, 32:] = 1
    want = dr.gather_grad32(g, idx, 2)
    with pytest.raises(AssertionError, match="differ in bits"):
        dr.check_bits(dr.gather_grad32(g, idx, 2, order="descending"), want, "reversed")
    up = _g((4, 12, 16), 9) * torch.tensor([1.0, 2.0 ** 20, -(2.0 ** 20), 3.0]).repeat(48)[:192].reshape(12, 16)
    with pytest.raises(AssertionError, match="differ in bits"):
        dr.check_bits(dr.upsample_backward32(up, 6, 8, True, order="descending"),
                      dr.upsample_backward32(up, 6, 8, True), "reversed upsample")


def test_pairwise_sum_is_rejected():
    g = dr.cancelling_terms(8, 64, 10)
    idx = torch.zeros((1, 64), dtype=torch.int32)
    with pytest.raises(AssertionError, match="differ in bits"):
        dr.check_bits(dr.pairwise_scatter(g, idx, 1), dr.gather_grad32(g, idx, 1), "pairwise")


def test_dropped_duplicate_slot_is_rejected():
    b, c, m, s, n = 2, 5, 40, 16, 100
    idx = _padded_balls(b, m, s, n, 11)
    g = _g((b, c, m, s), 12)
    r = dr.scatter64(g.reshape(b, c, -1), idx.reshape(b, -1), n)
    bad = dr.group_grad32(g, dr.drop_duplicate_slots(idx), n)
    with pytest.raises(AssertionError, match="outside the bound"):
        dr.check_bound(bad, r, "dropped duplicates")


@pytest.mark.parametrize("case", [(59, 80, 6, 6), (60, 80, 5, 8), (60, 80, 4, 8)])
def test_swapped_division_order_is_rejected(case):
    """kH / kW not a power of two (11 or 10 by 14, 12 by 10, 15 by 10): (g / kH) / kW and (g / kW) / kH differ in the
    last bit for many g"""
    ih, iw, oh, ow = case
    g = _g((3, oh, ow), 15)
    with pytest.raises(AssertionError, match="differ in bits"):
        dr.check_bits(dr.pool_backward32(g, ih, iw, div="swapped"), dr.pool_backward32(g, ih, iw), f"swapped {case}")


@pytest.mark.parametrize("case", [(7, 7, 3, 3), (80, 80, 6, 6), (59, 59, 6, 6)])
def test_floor_bin_end_is_rejected(case):
    ih, iw, oh, ow = case
    g = _g((3, oh, ow), 13).abs() + 0.5
    with pytest.raises(AssertionError, match="outside the bound"):
        dr.check_bound(dr.pool_backward32(g, ih, iw, end="floor"), dr.pool_backward64(g, ih, iw), f"floor {case}")


@pytest.mark.parametrize("case", [(6, 6, 60, 80, False), (6, 8, 12, 16, True), (3, 3, 60, 80, False)])
def test_wrong_align_corners_lambda_is_rejected(case):
    ih, iw, oh, ow, align = case
    g = _g((2, oh, ow), 14)
    with pytest.raises(AssertionError, match="outside the bound"):
        dr.check_bound(dr.upsample_backward32(g, ih, iw, align, lam="swapped"), dr.upsample_backward64(g, ih, iw, align),
                       f"swapped lambda {case}")


# ---- the workspace query ------------------------------------------------------------------------------------------
def _layout_bytes(b, n, slots):
    """pvn3d_ordered_grad_workspace_bytes restated: two key buffers (4 B, 8 B once b n >= 2^32), two slot buffers,
    b n + 1 run starts (8 B), and per 2048-pair tile 256 digit counts (4 B) and their scan (8 B); 256-byte pieces"""
    up = lambda x: -(-x // 256) * 256            # noqa: E731
    total, trash = b * slots, b * n
    ks = 8 if trash > 0xFFFFFFFF else 4
    tiles = -(-total // 2048)
    return 2 * up(ks * total) + 2 * up(4 * total) + up(8 * (trash + 1)) + up(4 * 256 * tiles) + up(8 * 256 * tiles)


@pytest.mark.parametrize("b,n,slots", [(24, 12288, 65536), (24, 2048, 1024 * 32), (24, 2048, 3 * 12288), (1, 1, 1),
                                       (1, 2 ** 21 + 1, 1024), (3, 2 ** 31 - 1, 7), (65535, 1, 2048)])
def test_workspace_query_is_host_arithmetic(b, n, slots):
    """the query needs no device (this test runs without one) and equals the layout, 64-bit keys included"""
    from pvn3d_b200 import _lib

    assert _lib.load().pvn3d_ordered_grad_workspace_bytes(b, n, slots) == _layout_bytes(b, n, slots)


def test_workspace_query_refusals():
    from pvn3d_b200 import _lib

    q = _lib.load().pvn3d_ordered_grad_workspace_bytes
    assert q(0, 10, 10) == 0 and q(1, 0, 10) == 0 and q(1, 10, 0) == 0
    assert q(65536, 10, 10) == 0 and q(1, 10, 2 ** 31) == 0
