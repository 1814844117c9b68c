"""The edge cases of csrc/normals.cu (tests/frame_input_cases.py) on the CPU: the float64 reference agrees with
plain brute force on every kNN case, every mutant differs from the reference on the cases that name it, and the
restated grid rule stays within its cell cap.  No GPU needed."""
import functools

import numpy as np
import pytest

import frame_input_cases as fc
import normals_ref as nr


@functools.lru_cache(maxsize=None)
def _knn_case(name):
    inputs = fc.KNN_CASES[name][0]()
    return inputs, [fc.knn_ref(inp) for inp in inputs]


@functools.lru_cache(maxsize=None)
def _sample(name):
    case = fc.sample_case(name)
    return case, fc.sample_ref(case, fc.sample_data(case))


# ---- the sampler ---------------------------------------------------------------------------------------------
def test_sample_cases_cover_the_edges():
    nvs = {}
    for name in fc.SAMPLE_CASES:
        case = fc.sample_case(name)
        nvs.setdefault(case["n"], set()).update(case["valid"].sum(1).tolist())
    for n in fc.SAMPLE_N:
        assert {400, 401, n + 1}.issubset(nvs[n]) and (n < 400 or {399, n - 1, n, 2 * n} <= nvs[n])
    combos = {(c["rgb_u8"], c["labels"], c["stride"]) for c in fc.SAMPLE_CASES.values()}
    assert len(combos) == 8 and len(fc.sample_case("b72")["valid"]) >= 70


@pytest.mark.parametrize("name", ["hw1025_n400", "hw3079_n50", "b72"])
def test_sample_rule_defaults_are_the_reference(name):
    case, ref = _sample(name)
    for f, v in enumerate(case["valid"]):
        c, o = fc.sample_rule(v, case["n"], case["seed"], f)
        assert o == ref["ok"][f] and np.array_equal(c, ref["choose"][f])


@pytest.mark.parametrize("mutant", fc.SAMPLE_MUTANTS)
def test_every_sampler_mutant_differs_on_some_case(mutant):
    assert any(fc.sample_mutant_differs(mutant, *(lambda c, r: (c, r["choose"], r["ok"]))(*_sample(name)))
               for name in fc.SAMPLE_CASES), mutant


# ---- the neighbour sets and normals ----------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(fc.KNN_CASES))
def test_knn_reference_is_brute_force(name):
    inputs, refs = _knn_case(name)
    for (ref, valid, q), want in zip(inputs, refs):
        for f in range(len(ref)):
            v = None if valid is None else valid[f]
            assert np.array_equal(want[f], nr.knn_brute(ref[f], q[f], v))
            if q.shape[1] * ref.shape[1] <= 2_000_000:
                assert np.array_equal(want[f], fc.knn_rule(ref[f], q[f], v))


@pytest.mark.parametrize("name", list(fc.KNN_CASES))
def test_case_rejects_its_mutants(name):
    inputs, refs = _knn_case(name)
    _, knn_mutants, normal_mutants = fc.KNN_CASES[name]
    for m in knn_mutants:
        assert any(not np.array_equal(fc.knn_mutant(m, inp), r) for inp, r in zip(inputs, refs)), m
    for inp, r in zip(inputs, refs):
        n, C, lam, curv = fc.normals_of(inp, r)
        assert fc.normal_faults(n, curv, C, lam, n, curv, inp[2].reshape(-1, 3))[0] == []
    for m in normal_mutants:
        assert any(fc.normal_mutant_faults(m, inp, r) for inp, r in zip(inputs, refs)), m


def test_every_mutant_is_named_by_a_case():
    assert {m for _, k, _ in fc.KNN_CASES.values() for m in k} == set(fc.KNN_MUTANTS)
    assert {m for _, _, n in fc.KNN_CASES.values() for m in n} == set(fc.NORMAL_MUTANTS)


def test_cases_hold_the_edges_they_name():
    ((ref, _, q),), _ = _knn_case("twins")
    assert (q[:, 0] == 0).all()
    for f in range(len(ref)):                                    # sub-ulp twins: float64 apart, float32 equal
        d = ref[f, :2].astype(np.float64)
        assert (d * d).sum(1)[0] > (d * d).sum(1)[1]
        d32 = ref[f, :2] * ref[f, :2]
        assert (d32[0, 0] + d32[0, 1]) + d32[0, 2] == (d32[1, 0] + d32[1, 1]) + d32[1, 2]
    ((ref, _, q),), (want,) = _knn_case("ties")
    d2 = nr.sqdist(q[0][:, None], ref[0][None])
    d50 = np.take_along_axis(d2, want[0][:, -1:], 1)
    assert ((d2 <= d50).sum(1) > 50).sum() > 100                  # exact ties at the 50th distance
    wrap = _knn_case("coincident_wrap")[0]
    assert np.unique(wrap[0][0][0], axis=0, return_counts=True)[1].max() >= 50
    assert np.unique(wrap[1][0][0], axis=0, return_counts=True)[1].max() == 31
    (ref, valid, _), = _knn_case("usable_counts")[0]
    usable = (valid & np.isfinite(ref).all(2)).sum(1)
    assert list(usable[:4]) == [49, 50, 51, 0] and usable[4] == ref.shape[1]


@pytest.mark.parametrize("name", list(fc.KNN_CASES))
def test_grid_rule_stays_within_its_cap(name):
    for ref, valid, _ in _knn_case(name)[0]:
        r = ref.shape[1]
        for f in range(len(ref)):
            v = None if valid is None else valid[f]
            lo, h, dims = fc.grid_rule(ref[f], v, r)
            assert np.prod(dims) <= 2 * r + 64
            assert np.frexp(h)[0] == 0.5                          # a power of two
            assert np.all(np.floor(lo / h) == lo / h)             # faces at exact multiples of the edge
            use = nr._usable(ref[f], v)
            if len(use):
                p = ref[f, use].astype(np.float64)
                assert (p >= lo).all() and (p < lo + dims * h).all()
