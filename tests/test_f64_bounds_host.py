"""The float64 references and bounds of tests/f64_bounds.py on the CPU: float32 emulations of the fused kernels'
arithmetic (TF32 operands, fp32 sums, the intermediates rounded to TF32 where the kernels round them) stay within the
bounds, and references that are wrong the way a kernel could be do not."""
import pytest
import torch

import f64_bounds as fb
from pvn3d_b200 import mlp

tf32 = mlp.tf32_round


def _layer(n, k, k_prev, g):
    return mlp.PackedLayer(torch.randn(n, k, generator=g) * k ** -0.5, torch.randn(n, generator=g) * 0.1, k_prev)


def _sa_operands(b, n, m, ns, c, n2, n3, seed):
    g = torch.Generator().manual_seed(seed)
    u = torch.randn(b * n, c, generator=g)
    v = torch.randn(b * m, c, generator=g) * 0.5
    idx = torch.randint(0, n, (b, m, ns), generator=g)
    rows_u = (torch.arange(b)[:, None, None] * n + idx).reshape(-1)
    rows_v = torch.arange(b * m).repeat_interleave(ns)
    l2 = _layer(n2, c, c, g)
    l3 = _layer(n3, n2, l2.n_pad, g)
    return u, v, rows_u, rows_v, l2, l3


def _sa_emulate(u, v, rows_u, rows_v, l2, l3, ns, round_out):
    """layers 2 and 3 + max-pool in float32 the way the kernels order them"""
    c = u.size(1)
    a2 = tf32(torch.relu(u[rows_u] - v[rows_v]))
    h = tf32(torch.relu(a2 @ l2.w[:, :c].t() + l2.bias))
    acc = (h @ l3.w[:, :h.size(1)].t()).view(-1, ns, l3.n_pad).amax(1)
    y = torch.relu(acc + l3.bias)
    return tf32(y) if round_out else y


@pytest.mark.parametrize("round_out", [False, True])
def test_sa_emulation_within_bound_and_mutations_outside(round_out):
    b, n, m, ns = 2, 300, 40, 16
    u, v, rows_u, rows_v, l2, l3 = _sa_operands(b, n, m, ns, 64, 96, 128, seed=1)
    got = _sa_emulate(u, v, rows_u, rows_v, l2, l3, ns, round_out)
    worst = fb.check(got, *fb.sa_scale(u, v, rows_u, rows_v, l2.w, l2.bias, l3.w, l3.bias, ns, round_out), "emulation")
    assert worst < 1.0
    w3 = l3.w.clone()
    w3[:, 64:] = 0                                                  # the last layer-3 K chunk dropped
    b3 = l3.bias.clone()
    b3[:l3.n] = b3[:l3.n].roll(1)                                   # b3 rolled by one column
    rows_prev = rows_u.clone()
    rows_prev[m * ns:(m + 1) * ns] -= n                             # one centre's neighbours from the previous frame
    for name, (ru, w, bias) in [("last k chunk dropped", (rows_u, w3, l3.bias)), ("b3 rolled", (rows_u, l3.w, b3)),
                                ("previous frame", (rows_prev, l3.w, l3.bias))]:
        with pytest.raises(AssertionError, match="outside the bound"):
            fb.check(got, *fb.sa_scale(u, v, ru, rows_v, l2.w, l2.bias, w, bias, ns, round_out), name)


def _fma32(a, b, c):
    """fp32 fma: the exact a*b (a float64 product of float32 values) plus c, rounded once more to float32"""
    return (a.double() * b.double() + c.double()).float()


def _interp32(p, rows, w):
    """fma(p3,w3, fma(p1,w1, p2*w2)) in float32, as the kernels contract it"""
    p1, p2, p3 = (p[rows[:, t]] for t in range(3))
    w1, w2, w3 = (w[:, t:t + 1] for t in range(3))
    return _fma32(p3, w3, _fma32(p1, w1, p2 * w2))


def test_interpolation_bound_holds_for_the_fp32_fma_chain():
    g = torch.Generator().manual_seed(2)
    p = torch.randn(500, 64, generator=g) * torch.logspace(-3, 3, 64)
    rows = torch.randint(0, 500, (4000, 3), generator=g)
    w = torch.rand(4000, 3, generator=g) + 0.01
    w = w / w.sum(1, keepdim=True)
    fb.check(_interp32(p, rows, w), *fb.interp(p, rows, w), "fma chain")


def test_fp_module_emulation_within_bound():
    g = torch.Generator().manual_seed(3)
    rows, m, c2, c1 = 700, 129, 80, 52
    known = torch.randn(m, c2, generator=g)
    skip = torch.randn(rows, 60, generator=g)
    nn_rows = torch.randint(0, m, (rows, 3), generator=g)
    nn_w = torch.rand(rows, 3, generator=g) + 0.05
    nn_w = nn_w / nn_w.sum(1, keepdim=True)
    l1 = _layer(256, c2 + c1, None, g)
    l2 = _layer(384, 256, l1.n_pad, g)
    x = torch.cat([tf32(_interp32(known, nn_rows, nn_w)), tf32(skip[:, :c1].contiguous())], 1)
    h = tf32(torch.relu(x @ l1.w[:, :c2 + c1].t() + l1.bias))
    got = torch.relu(h @ l2.w[:, :256].t() + l2.bias)
    fb.check(got, *fb.fp_module(known, nn_rows, nn_w, skip, c1, l1.w, l1.bias, l2.w, l2.bias, False), "fp2 emulation")
    with pytest.raises(AssertionError, match="outside the bound"):
        fb.check(got, *fb.fp_module(known, nn_rows, nn_w[:, [1, 0, 2]], skip, c1, l1.w, l1.bias, l2.w, l2.bias, False),
                 "weights 1 and 2 swapped")


def test_fp1_module_emulation_within_bound():
    g = torch.Generator().manual_seed(4)
    rows, m = 900, 200
    p = torch.randn(m, 128, generator=g) * 0.5
    table = tf32(torch.cat([torch.randn(rows, 12, generator=g), torch.zeros(rows, 20)], 1))
    nn_rows = torch.randint(0, m, (rows, 3), generator=g)
    nn_w = torch.rand(rows, 3, generator=g) + 0.05
    nn_w = nn_w / nn_w.sum(1, keepdim=True)
    ls = _layer(128, 12, None, g)
    l2 = _layer(128, 128, ls.n_pad, g)
    s = table @ ls.w[:, :32].t() + ls.bias
    a = tf32(torch.relu(_interp32(p, nn_rows, nn_w) + s))
    got = tf32(torch.relu(a @ l2.w.t() + l2.bias))
    fb.check(got, *fb.fp1_module(p, nn_rows, nn_w, table, ls.w, ls.bias, l2.w, l2.bias, True), "fp1 emulation")
    with pytest.raises(AssertionError, match="outside the bound"):
        fb.check(got, *fb.fp1_module(p, nn_rows, nn_w, table, ls.w, torch.zeros(128), l2.w, l2.bias, True), "b_s omitted")


def test_check_holds_zero_bounds_to_equality_and_rejects_nan():
    ref = torch.tensor([[1.0, 0.0]], dtype=torch.float64)
    bound = torch.tensor([[1e-3, 0.0]], dtype=torch.float64)
    assert fb.check(torch.tensor([[1.0005, 0.0]]), ref, bound) == pytest.approx(0.5, rel=1e-3)
    with pytest.raises(AssertionError, match="outside the bound"):
        fb.check(torch.tensor([[1.0, 1e-30]]), ref, bound)
    with pytest.raises(AssertionError, match="outside the bound"):
        fb.check(torch.tensor([[float("nan"), 0.0]]), ref, bound)
