"""tests/grad_ref.py on the CPU: the float64 references of the PointNet++ gradient ops against plain loops, the
gamma_k bound against float32 sums in many orders, the exact cases, and every mutant rejected where it should be."""
import numpy as np
import pytest
import torch

import grad_ref as gr

F32 = np.float32


def _loop_scatter(terms, idx, n):
    b, c, j = terms.shape
    out = np.zeros((b, c, n))
    for f in range(b):
        for l in range(c):
            for s in range(j):
                out[f, l, idx[f, s]] += float(terms[f, l, s])
    return out


def test_references_equal_a_plain_loop():
    rng = np.random.default_rng(0)
    b, c, n, m, s = 2, 3, 11, 5, 4
    g = rng.normal(size=(b, c, m, s)).astype(F32)
    idx = rng.integers(0, n, size=(b, m, s)).astype(np.int32)
    r = gr.group_grad(torch.from_numpy(g), torch.from_numpy(idx), n)
    assert np.array_equal(r.ref.numpy(), _loop_scatter(g.reshape(b, c, -1).astype(np.float64), idx.reshape(b, -1), n))
    assert np.array_equal(r.k[:, 0].numpy(), np.stack([np.bincount(i.reshape(-1), minlength=n) for i in idx]))
    assert np.allclose(r.s.numpy(), _loop_scatter(np.abs(g.reshape(b, c, -1)).astype(np.float64), idx.reshape(b, -1), n),
                       rtol=1e-15, atol=0)

    g2 = rng.normal(size=(b, c, m)).astype(F32)
    idx2 = rng.integers(0, n, size=(b, m)).astype(np.int32)
    r2 = gr.gather_grad(torch.from_numpy(g2), torch.from_numpy(idx2), n)
    assert np.array_equal(r2.ref.numpy(), _loop_scatter(g2.astype(np.float64), idx2, n))

    gi = rng.normal(size=(b, c, n)).astype(F32)
    ii = rng.integers(0, m, size=(b, n, 3)).astype(np.int32)
    w = rng.uniform(size=(b, n, 3)).astype(F32)
    ri = gr.interp_grad(torch.from_numpy(gi), torch.from_numpy(ii), torch.from_numpy(w), m)
    want = np.zeros((b, c, m))
    for f in range(b):
        for l in range(c):
            for j in range(n):
                for t in range(3):
                    want[f, l, ii[f, j, t]] += float(gi[f, l, j]) * float(w[f, j, t])   # exact: 24 + 24 bits
    assert np.allclose(ri.ref.numpy(), want, rtol=1e-15, atol=1e-300)
    assert np.array_equal(ri.k[:, 0].numpy(), np.stack([np.bincount(i.reshape(-1), minlength=m) for i in ii]))


def test_k1_reference_is_the_float32_product():
    """k = 1 of the interpolation: the float64 reference rounded to float32 is torch's float32 product g*w (a -0.0
    product becomes +0.0 on the memset's zero)"""
    rng = np.random.default_rng(1)
    b, c, n, m = 1, 4, 9, 27
    g = torch.from_numpy(rng.normal(size=(b, c, n)).astype(F32))
    g[0, 0, 0] = -1.0
    idx = torch.arange(n * 3, dtype=torch.int32).reshape(b, n, 3)          # every known point hit once
    w = torch.from_numpy(rng.uniform(size=(b, n, 3)).astype(F32))
    w[0, 0, 0] = 0.0                                                     # -1 * 0 = -0.0
    r = gr.interp_grad(g, idx, w, m)
    assert bool((r.k == 1).all())
    prod = (g[..., None] * w[:, None]).reshape(b, c, m)
    assert torch.equal(r.ref.float(), prod)                              # values (-0.0 == +0.0)
    got = (torch.zeros_like(prod) + prod)                                # what one atomic add onto the zero leaves
    gr.check(got, r, "interp k=1")
    assert gr._bits(got)[0, 0, 0] == 0


def _orders(terms, idx, n, orders, rng):
    """float32 sequential scatter-adds of terms [C,J] (idx [J]) in `orders` random orders -> [orders, C, n]"""
    c, j = terms.shape
    out = np.zeros((orders, c, n), F32)
    for o in range(orders):
        p = rng.permutation(j)
        tp, ip = terms[:, p], idx[p]
        for a in range(n):
            sel = tp[:, ip == a]
            if sel.shape[1]:
                out[o, :, a] = np.add.accumulate(sel, axis=1, dtype=F32)[:, -1]
    return out


@pytest.mark.parametrize("op", ["gather", "interp"])
def test_float32_sums_in_any_order_stay_within_the_bound(op):
    rng = np.random.default_rng(2)
    c, j, n = 3, 6000, 4                                  # k ~ 1500 (gather) / 4500 (interp) per element, mixed signs
    g = (rng.normal(size=(1, c, j)) * np.exp(rng.uniform(-3, 3, size=(1, c, j)))).astype(F32)
    if op == "gather":
        idx = rng.integers(0, n, size=(1, j)).astype(np.int32)
        r = gr.gather_grad(torch.from_numpy(g), torch.from_numpy(idx), n)
        terms, flat = g[0], idx[0]
    else:
        idx = rng.integers(0, n, size=(1, j, 3)).astype(np.int32)
        w = rng.uniform(size=(1, j, 3)).astype(F32)
        r = gr.interp_grad(torch.from_numpy(g), torch.from_numpy(idx), torch.from_numpy(w), n)
        terms = (g[0][..., None] * w[0][None]).astype(F32).reshape(c, -1)     # fl32(g*w), as the kernel
        flat = idx[0].reshape(-1)
    assert int(r.k.min()) > 1000
    got = _orders(terms, flat, n, 60, rng)
    worst = max(gr.check(torch.from_numpy(o[None]), r, f"{op} order {i}") for i, o in enumerate(got))
    assert 0 < worst < 1                                  # the orders really differ from the exact sum


def test_integer_terms_sum_exactly_in_any_order():
    """integer g and weights in multiples of 1/8: every partial sum is a multiple of 1/8 below 2^21, so float32 holds
    it exactly and any order gives the float64 sum -- check(exact=True) passes; a float g in the same orders does not"""
    rng = np.random.default_rng(3)
    c, j, n = 2, 5000, 3
    g = rng.integers(-8, 9, size=(1, c, j)).astype(F32)
    idx = rng.integers(0, n, size=(1, j, 3)).astype(np.int32)
    w = (rng.integers(0, 9, size=(1, j, 3)) / 8).astype(F32)
    r = gr.interp_grad(torch.from_numpy(g), torch.from_numpy(idx), torch.from_numpy(w), n)
    assert float(r.s.max()) * 8 < 2 ** 24
    terms = (g[0][..., None] * w[0][None]).astype(F32).reshape(c, -1)
    for i, o in enumerate(_orders(terms, idx[0].reshape(-1), n, 20, rng)):
        gr.check(torch.from_numpy(o[None]), r, f"integer order {i}", exact=True)
    gf = g + rng.normal(size=g.shape).astype(F32) * F32(1e-3)
    rf = gr.interp_grad(torch.from_numpy(gf), torch.from_numpy(idx), torch.from_numpy(w), n)
    tf = (gf[0][..., None] * w[0][None]).astype(F32).reshape(c, -1)
    got = _orders(tf, idx[0].reshape(-1), n, 5, rng)
    with pytest.raises(AssertionError, match="outside the bound"):
        for o in got:
            gr.check(torch.from_numpy(o[None]), rf, "float g, exact", exact=True)


def test_exact_cases_are_demanded():
    rng = np.random.default_rng(4)
    g = torch.from_numpy(rng.normal(size=(1, 2, 3)).astype(F32))
    idx = torch.tensor([[0, 2, 2]], dtype=torch.int32)                   # k = 1, 0, 2
    r = gr.gather_grad(g, idx, 3)
    good = r.ref.float()
    gr.check(good, r, "exact")
    neg0 = good.clone()
    neg0[:, :, 1] = -0.0                                                 # k = 0 must be +0.0, not -0.0
    with pytest.raises(AssertionError, match="outside the bound"):
        gr.check(neg0, r, "-0")
    off = good.clone()
    off[0, 0, 0] = float(np.nextafter(F32(off[0, 0, 0]), F32(np.inf)))      # k = 1 one ulp off: inside gamma_1 S, not exact
    with pytest.raises(AssertionError, match="outside the bound"):
        gr.check(off, r, "k=1 ulp")
    nan = good.clone()
    nan[0, 1, 2] = float("nan")
    with pytest.raises(AssertionError, match="outside the bound"):
        gr.check(nan, r, "nan")


def _ball_like(rng, b, m, s, n):
    """rows of a ball query: a few hits, the rest padded with the first hit, some empty rows of zeros"""
    idx = np.zeros((b, m, s), np.int32)
    for f in range(b):
        for j in range(m):
            hits = np.sort(rng.choice(n, size=int(rng.integers(0, s + 1)), replace=False))
            if len(hits):
                idx[f, j] = hits[0]
                idx[f, j, :len(hits)] = hits
    return idx


def test_mutants_are_rejected():
    rng = np.random.default_rng(5)
    b, c, m, s, n = 3, 7, 64, 16, 300
    idx = torch.from_numpy(_ball_like(rng, b, m, s, n))
    g = torch.from_numpy(rng.normal(size=(b, c, m, s)).astype(F32))
    r = gr.group_grad(g, idx, n)
    gr.check(r.ref.float(), r, "group, the reference itself")
    muts = {
        "dedup": gr.mut_group_dedup(g, idx, n),
        "frame0": gr.mut_frames(r, "frame0"),
        "shift": gr.mut_frames(r, "shift"),
        "last channel": gr.mut_drop_channels(r, [c - 1]),
        "last slice": gr.mut_drop_channels(r, range(gr.channel_slices(c, 1, 4) - 1, c, gr.channel_slices(c, 1, 4))),
        "drop one": gr.mut_drop_one(g.reshape(b, c, -1), idx.reshape(b, -1), r),
    }
    for name, got in muts.items():
        with pytest.raises(AssertionError, match="outside the bound"):
            gr.check(got, r, name)

    nn = torch.from_numpy(rng.integers(0, m, size=(b, n, 3)).astype(np.int32))
    w = torch.from_numpy(rng.uniform(size=(b, n, 3)).astype(F32))
    gi = torch.from_numpy(rng.normal(size=(b, c, n)).astype(F32))
    ri = gr.interp_grad(gi, nn, w, m)
    gr.check(ri.ref.float(), ri, "interp, the reference itself")
    for name, got in {"swapped weights": gr.interp_grad(gi, nn, gr.mut_swap_nn_weights(w), m).ref.float(),
                      "reference wrapper": torch.from_numpy(gr.mut_reference_wrapper(gi.numpy(), nn.numpy(), w.numpy(),
                                                                                     m)),
                      "drop one": gr.mut_drop_one(gr.interp_terms(gi, w), nn.reshape(b, -1), ri)}.items():
        with pytest.raises(AssertionError, match="outside the bound"):
            gr.check(got, ri, name)


def test_channel_slices_restatement():
    assert gr.channel_slices(96, 128 * 24, 132) == 1
    assert gr.channel_slices(1024, 1, 132) == 528
    assert gr.channel_slices(5, 1, 132) == 5
    assert gr.channel_slices(300, 7, 132) == 76
