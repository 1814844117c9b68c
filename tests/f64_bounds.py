"""Float64 references of the fused shared-MLP kernels with an element-wise error bound (test infrastructure, no
conftest).  Everything is float64 on whatever device the operands live on.

A reference value comes with a bound on |kernel - reference| that is built stage by stage:

  * accumulation: a layer act(A . W^T + b) on TF32 operands accumulates in fp32 -> 1e-5 of S = |A| . |W|^T + |b| (as
    the bf16 tests allow; the fp32 error of a K <= 1024 sum is ~100x smaller, so 1e-5 only matters where the sum
    cancels);
  * operand uncertainty: where the kernel rounds an intermediate to TF32 and the reference cannot reproduce the value
    before rounding bit for bit (an fp32-accumulated layer, the fp32 fma chain of the interpolation), the reference
    rounds its own value with mlp.tf32_round (nearest, ties away, as cvt.rna) and carries delta = eps_upstream +
    2^-10 |ref| per element: two roundings of values within eps of each other, each within half a TF32 ulp
    (2^-11 of the binade, and |ref| is never below its binade).  The next layer's bound gains delta . |W|^T;
  * exact stages: tf32(relu(U[idx] - V)) is one fp32 subtraction of the kernels' own U and V, a ReLU and a rounding --
    reproduced exactly, delta = 0;
  * bias, ReLU and max-pool are 1-Lipschitz: the bound passes through them (max-pool: the largest row bound of the
    window).  A TF32-rounded output adds 2^-10 |ref|;
  * interpolation fma(p3,w3, fma(p1,w1, p2*w2)): three fp32 roundings, <= 3 * 2^-24 sum_t |w_t p_t|, carried as
    2^-22 sum_t |w_t p_t| (the spare 2^-24 covers the reference's own float64 -> float32 step before rounding).

The slack of the rounding terms (the 2^-24 |x| of the reference's float64 -> float32 step, the 2^-11 eps of a kernel
value rounded from x + eps) is far inside the 1e-5 S of the layer that produced x, since S >= |x|.
"""
from __future__ import annotations

import torch

from pvn3d_b200.mlp import tf32_round

ACC = 1e-5              # fp32 accumulation allowance, relative to |A| . |W|^T + |b|
TF32_ROUND = 2.0 ** -10  # two TF32 roundings of nearby values: one TF32 ulp relative to the rounded value
INTERP = 2.0 ** -22     # the fp32 fma chain of the three-point interpolation, relative to sum_t |w_t p_t|
F32 = 2.0 ** -24        # one fp32 rounding, relative


def tf32(x: torch.Tensor) -> torch.Tensor:
    """float64 -> the TF32 value the reference rounds it to (via float32, as the kernels round fp32 values)"""
    return tf32_round(x.float()).double()


def dense(a: torch.Tensor, w: torch.Tensor, b: torch.Tensor, delta: torch.Tensor | None = None, relu: bool = True):
    """one layer on TF32 operands: a [rows, K] (the values the kernel multiplies), w [N, K], b [N] or [rows, N] ->
    (act(a . w^T + b), ACC (|a| . |w|^T + |b|) + delta . |w|^T), float64"""
    a, w, b = a.double(), w.double(), b.double()
    ref = a @ w.t() + b
    wa = w.abs().t()
    bound = ACC * (a.abs() @ wa + b.abs())
    if delta is not None:
        bound = bound + delta @ wa
    return (ref.clamp_min(0) if relu else ref), bound


def round_tf32(ref: torch.Tensor, bound: torch.Tensor):
    """a value the kernel rounds to TF32 (an intermediate or a ROUND_OUT store): the reference rounds its own value and
    the bound gains one TF32 ulp of it"""
    r = tf32(ref)
    return r, bound + TF32_ROUND * r.abs()


def max_pool(ref: torch.Tensor, bound: torch.Tensor, pool: int):
    """max over consecutive groups of `pool` rows: the reference's maximum, the largest row bound of the window"""
    n = ref.size(-1)
    return ref.view(-1, pool, n).amax(1), bound.view(-1, pool, n).amax(1)


def group_sum(ref: torch.Tensor, bound: torch.Tensor, group: int):
    """sums over consecutive groups of `group` rows (a partial last group sums what there is): errors add"""
    rows, n = ref.shape
    pad = -rows % group
    ref = torch.nn.functional.pad(ref, (0, 0, 0, pad)).view(-1, group, n).sum(1)
    bound = torch.nn.functional.pad(bound, (0, 0, 0, pad)).view(-1, group, n).sum(1)
    return ref, bound


def interp(p: torch.Tensor, rows: torch.Tensor, w: torch.Tensor):
    """three-point interpolation sum_t w_t p[rows_t]: p [M, C], rows [R, 3] (int64, rows of p), w [R, 3] ->
    (reference [R, C], INTERP sum_t |w_t p[rows_t]|)"""
    terms = p.double()[rows] * w.double()[..., None]          # [R, 3, C]
    return terms.sum(1), INTERP * terms.abs().sum(1)


def check(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, what: str = "") -> float:
    """assert |got - ref| <= bound everywhere (where the bound is 0 -- zero-padded columns -- got must equal ref);
    returns and prints the worst |got - ref| / bound"""
    assert got.shape == ref.shape == bound.shape, (what, tuple(got.shape), tuple(ref.shape), tuple(bound.shape))
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)                                     # NaN in got counts as outside
    pos = bound > 0
    worst = float((err[pos] / bound[pos]).max()) if bool(pos.any()) else 0.0
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        idx = tuple(int(x) for x in torch.unravel_index(torch.tensor(i), bad.shape))
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the bound, first at {idx}: "
                             f"got {float(got[idx])!r} ref {float(ref[idx])!r} bound {float(bound[idx]):.3g}; "
                             f"worst |got - ref| / bound {worst:.3g}")
    print(f"{what}: worst |got - ref| / bound {worst:.3g}")
    return worst


# ---- the fused kernels' operations -----------------------------------------------------------------------------------


def sa_scale(u, v, rows_u, rows_v, w2, b2, w3, b3, ns: int, round_out: bool):
    """layers 2 and 3 of a factored SA scale + max-pool (pvn3d_mlp_sa_fact2 / _sa_fact2w): u [*, C], v [*, C] the f32
    tables the kernels read, rows_u / rows_v [rows] (int64) the U and V row of every grouped row (centre-major, ns per
    centre), w2 [N2, >= C], w3 [N3, >= N2] the packed TF32 weights -> (reference, bound) [rows / ns, N3]"""
    c = u.size(-1)
    a2 = tf32_round(torch.relu(u[rows_u] - v[rows_v])).double()      # the kernels' own fp32 arithmetic: exact
    h, e = round_tf32(*dense(a2, w2[:, :c], b2))
    y, e = dense(h, w3[:, :h.size(1)], b3, e)
    y, e = max_pool(y, e, ns)
    return round_tf32(y, e) if round_out else (y, e)


def fp_module(known, nn_rows, nn_w, skip, c1: int, w1, b1, w2, b2, round_out: bool):
    """both layers of an FP2-FP4 module (pvn3d_mlp_fp2): known [M, c2] f32, nn_rows [R, 3] (int64 rows of known),
    nn_w [R, 3], skip [R, >= c1] f32, w1 [N1, >= c2 + c1], w2 [N2, >= N1] packed TF32 -> (reference, bound) [R, N2]"""
    c2 = known.size(-1)
    x, ex = round_tf32(*interp(known, nn_rows, nn_w))
    s = tf32_round(skip[:, :c1].contiguous()).double()
    a = torch.cat([x, s], 1)
    ea = torch.cat([ex, torch.zeros_like(s)], 1)
    h, e = round_tf32(*dense(a, w1[:, :c2 + c1], b1, ea))
    y, e = dense(h, w2[:, :h.size(1)], b2, e)
    return round_tf32(y, e) if round_out else (y, e)


def fp1_module(p, nn_rows, nn_w, table, ws, bs, w2, b2, round_out: bool):
    """the skip term and second layer of the factored FP1 module (pvn3d_mlp_fp_fact2 / _rows): p [M, C] f32 (P = W1k .
    known), nn_rows / nn_w [R, 3], table [R, K] the TF32 factor-table rows, ws [C, >= K] + bs [C] the skip layer,
    w2 [N2, >= C] -> (reference, bound) [R, N2], point-major: relu(tf32(relu(interp(P) + table . ws^T + bs)) . w2^T + b2)"""
    s, es = dense(table, ws[:, :table.size(1)], bs, relu=False)
    x, ex = interp(p, nn_rows, nn_w)
    # the kernel adds the fp32 interpolation to fl(S + b_s): two more fp32 roundings before the TF32 one
    a, e = round_tf32((x + s).clamp_min(0), ex + es + 2 * F32 * (x.abs() + s.abs()))
    y, e = dense(a, w2[:, :a.size(1)], b2, e)
    return round_tf32(y, e) if round_out else (y, e)
