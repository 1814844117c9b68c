"""The references, builders and mutants of tests/geo_ref.py checked on the host: a reference that is wrong, or a
mutant that equals the oracle on the inputs it is used with, would make the GPU checks prove nothing."""
import numpy as np
import pytest

import geo_ref as G
import pn2_edge_cases as C
from oracle import pn2

F32 = np.float32


def test_weights_ref_hand_rows_and_f64_bound():
    inf = np.inf
    w = G.weights_ref(np.array([[0, 0, 0], [0, 0, inf], [0, inf, inf], [1e-4, inf, inf], [inf, inf, inf]], np.float32))
    assert np.array_equal(w[0], np.full(3, F32(1) / F32(3)))            # three coincident known points: 1/3 each
    assert w[1].tolist() == [0.5, 0.5, 0.0] and w[2].tolist() == [1.0, 0.0, 0.0] and w[3].tolist() == [1.0, 0.0, 0.0]
    assert np.isnan(w[4]).all()                                         # 0 / 0, as torch gives
    r0 = F32(1) / F32(1e-8)
    assert abs(float(r0) - 1e8) < 10                                    # "1e8 before normalisation"
    one_zero = G.weights_ref(np.array([[0, 1e-4, 4e-4]], np.float32))[0]
    assert one_zero[0] == F32(r0 / ((r0 + F32(1) / (F32(0.01) + G.EPS)) + F32(1) / (F32(0.02) + G.EPS)))
    d2 = C.weight_inputs(100000, 1)
    assert (d2 == 0).any() and np.isinf(d2).any() and ((d2 > 0) & (d2 < 1.2e-38)).any()
    w32, w64 = G.weights_ref(d2), G.weights_f64(d2)
    assert G.weights_err_over_bound(w32, w64) <= 1.0
    assert G.weights_err_over_bound(G.mut_weights_no_eps(np.full((4, 3), 1e-14, np.float32) * [1, 2, 3]),
                                    G.weights_f64(np.full((4, 3), 1e-14, np.float32) * [1, 2, 3])) > 1e3
    assert not G.same_bits(G.mut_weights_no_eps(d2), w32)


def test_factor_table_and_centre_term_refs_on_hand_rows():
    # 1 + 2^-11 is a tie in TF32: rounds AWAY (1 + 2^-10); 1 + 2^-12 rounds down, and lo keeps what hi dropped
    x = np.array([[1 + 2.0 ** -11, 1 + 2.0 ** -12, -(1 + 2.0 ** -11)]], np.float32)
    f = np.array([[3.0, 1 + 2.0 ** -11, 7.0]], np.float32)              # ldf 3 > c_feat 2
    tab = G.factor_table_ref(x, f, 2, 32)
    assert tab[0, :2].tolist() == [3.0, 1 + 2.0 ** -10]
    assert tab[0, 2:5].tolist() == [1 + 2.0 ** -10, 1.0, -(1 + 2.0 ** -10)]
    assert tab[0, 5:8].tolist() == [-(2.0 ** -11), 2.0 ** -12, 2.0 ** -11]
    assert not tab[0, 8:].any()
    for cloud in (G.raster_cloud(1, 2048, 3)[0], G.far(G.raster_cloud(1, 2048, 3))[0], G.tiny(G.raster_cloud(1, 2048, 3))[0]):
        t = G.factor_table_ref(cloud, None, 0, 32)
        assert G.split_rel_err(cloud, t, 0) <= 2.0 ** -21
        assert G.split_rel_err(cloud, G.mut_table_no_lo(t, 0), 0) > 2.0 ** -14
    v, bound = G.centre_term_f64(np.array([[1.0, 2.0, 3.0]]), np.array([[0.5, -1.0, 2.0], [0, 0, 0]]), np.array([0.25, 1.0]))
    assert v.tolist() == [[4.25, -1.0]] and np.allclose(bound, 1e-6 * np.array([[8.75, 1.0]]))


def test_radius_shell_straddles_r2_in_the_last_bits():
    radii = (0.0175, 0.025)
    cloud, centres, rows = G.radius_shell(12288, 256, radii, 50)
    d2 = pn2.sqdist(centres[0, rows], cloud[0])
    for r in radii:
        r2 = F32(r) * F32(r)
        near = np.abs(d2.astype(np.float64) - float(r2)) <= 40 * float(np.spacing(r2))
        assert (d2[near] < r2).any() and (d2[near] == r2).any() and (d2[near] > r2).any()
        assert near.sum(1).min() >= 2 * len(G.SHELL_KS)
    # tight boxes: a 128-point box of the x-sorted cloud is a small fraction of the slab in x
    xs = cloud[0, :, 0].reshape(-1, 128)
    assert np.median(xs.max(1) - xs.min(1)) < 0.05


def test_builders_are_seeded_and_have_ties():
    a, b = C._tie_cloud(2, 1000, 5), C._tie_cloud(2, 1000, 5)
    assert np.array_equal(a, b)
    assert len(np.unique(G.bits(a[0]), axis=0)) < 1000
    assert not np.array_equal(a[0], a[1])
    s = G.sorted_cloud(a, 1)
    assert (np.diff(s[..., 1], axis=1) >= 0).all()
    assert np.array_equal(np.sort(G.shuffled(a, 1)[0], 0), np.sort(a[0], 0))


@pytest.mark.parametrize("name", [n for n, (_, mu) in C.FPS_CASES.items() if mu and n != "bench_stress"])
def test_fps_mutants_differ_from_oracle(name):
    build, names = C.FPS_CASES[name]
    inputs = build()
    refs = [pn2.furthest_point_sampling(x, m) for x, m in inputs]
    for nm, mu in C.fps_mutants(names, inputs, refs).items():
        assert C.some_differ(refs, mu), nm


@pytest.mark.parametrize("name", [n for n in C.BALL_CASES if n not in ("raster_49152", "n_131072", "n_131273_blk256")])
def test_ball_mutants_differ_from_oracle(name):
    build, names = C.BALL_CASES[name]
    inputs = build()
    refs = C.ball_refs(inputs)
    for nm, mu in C.ball_mutants(names, inputs, refs).items():
        assert C.some_differ(refs, mu), nm
    if name == "shell":          # the numpy row restatement the `<=` mutant is built from agrees with the oracle
        x, c, radii, nss = inputs[0]
        for ref, r, ns in zip(refs[0], radii, nss):
            assert np.array_equal(G.ball_rows_np(c[0, :32], x[0], float(F32(r)), ns), ref[0, :32])


@pytest.mark.parametrize("name", [n for n in C.NN_CASES if n != "bench_49152x2048"])
def test_three_nn_mutants_differ_from_oracle(name):
    build, names = C.NN_CASES[name]
    inputs = build()
    refs = [pn2.three_nn(u, k) for u, k in inputs]
    for nm, mu in C.nn_mutants(names, inputs, refs).items():
        assert C.some_differ([r[1] for r in refs], mu), nm


def test_fps_lowest_index_is_the_oracle_without_ties():
    x = G.uniform_cloud(1, 700, 9)
    assert np.array_equal(G.fps_lowest_index(x[0], 40), pn2.furthest_point_sampling(x, 40)[0])
