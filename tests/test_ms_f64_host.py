"""The float64 mean-shift and Kabsch references of tests/ms_f64.py against what the reference recorded (CPU only).

The GPU checks of tests/test_meanshift_f64_gpu.py and tests/test_kabsch_f64_gpu.py are only as good as these
references, so they are pinned here to the reference's own outputs: on every recorded mean-shift case T is within
+-1 of the recorded iteration count, the labels are exact and the centre is within 1e-5 relative; the Kabsch
reference reproduces every recorded best_fit_transform.
"""
import os

import numpy as np
import pytest
import torch

import ms_f64

CASES = ["tight", "outl10", "outl30", "two", "wide", "bw002", "bw016", "single", "pair_far", "n1200"]


def _case(golden_dir, name):
    if name == "sym2":
        z = np.load(os.path.join(golden_dir, "ms_big.npz"))
        n = len(z["sym2_A"])
        return z["sym2_A"], float(z["sym2_bw"]), np.unpackbits(z["sym2_labels"])[:n].astype(bool), z["sym2_ctr"], \
            int(z["sym2_iters"])
    z = np.load(os.path.join(golden_dir, "ms_cases.npz"))
    return z[f"{name}_A"], float(z[f"{name}_bw"]), z[f"{name}_labels"], z[f"{name}_ctr"], int(z[f"{name}_iters"])


@pytest.mark.parametrize("name", CASES + ["sym2"])
def test_f64_reference_matches_recorded_fits(golden_dir, name):
    A, bw, labels, ctr, iters = _case(golden_dir, name)
    ref = ms_f64.reference([A], bw, 300, torch.device("cpu"))[0]
    assert np.array_equal(ref["labels"], labels.astype(bool)), "labels must be bit-exact"
    assert abs(ref["T"] - iters) <= 1, (ref["T"], iters)
    c = ref["traj"][ref["T"]]
    assert np.linalg.norm(c - ctr) <= 1e-5 * np.linalg.norm(ctr), (c, ctr)
    # the star's trajectory starts at its input point
    assert np.array_equal(ref["traj"][0], A[ref["max_idx"]].astype(np.float64))


def test_f64_batching_does_not_change_a_fit(golden_dir):
    """fits batched together (padded to the largest) give what each gives alone"""
    clouds = [_case(golden_dir, n)[0] for n in ("tight", "two", "wide", "bw002")]
    bw = 0.08
    mi = [ms_f64.exact_part(A, bw)[1] for A in clouds]
    together = ms_f64.iterate_f64(clouds, bw, 300, mi, torch.device("cpu"))
    for A, m, r in zip(clouds, mi, together):
        alone = ms_f64.iterate_f64([A], bw, 300, [m], torch.device("cpu"))[0]
        assert alone["T"] == r["T"]
        assert np.allclose(alone["traj"], r["traj"], rtol=0, atol=1e-12)


def test_f64_max_iter_and_empty():
    A = np.array([[0.1, 0.2, 0.9], [0.13, 0.2, 0.9], [0.5, 0.2, 0.9]], np.float32)
    for max_iter in (0, 1, 5):
        r = ms_f64.reference([A], 0.08, max_iter, torch.device("cpu"))[0]
        assert r["T"] <= max_iter + 1 and len(r["traj"]) == r["T"] + 2
    assert ms_f64.reference([A], 0.08, 0, torch.device("cpu"))[0]["T"] == 1
    e = ms_f64.reference([np.zeros((0, 3), np.float32)], 0.08, 300, torch.device("cpu"))[0]
    assert e["max_idx"] == -1 and "T" not in e


def test_kabsch_reference_matches_recorded_transforms(golden_dir):
    z = np.load(os.path.join(golden_dir, "bft_cases.npz"))
    for a, b, tref in zip(z["A"], z["B"], z["T"]):
        R, t, _ = ms_f64.kabsch_f64(a, b)
        assert np.linalg.norm(R - tref[:, :3]) <= 1e-5 and np.linalg.norm(t - tref[:, 3]) <= 1e-5 * max(1.0, np.linalg.norm(tref[:, 3]))
        assert abs(np.linalg.det(R) - 1.0) < 1e-12


def test_wrong_kabsch_reference_is_caught():
    """without the reflection fix a reflected target gives det -1, which the check rejects"""
    rng = np.random.default_rng(0)
    A = rng.normal(size=(9, 3))
    B = A * np.array([1.0, 1.0, -1.0])
    R, _, _ = ms_f64.kabsch_f64(A, B, reflection_fix=False)
    assert np.linalg.det(R) < 0
    R, _, _ = ms_f64.kabsch_f64(A, B)
    assert np.linalg.det(R) > 0
