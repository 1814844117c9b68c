"""The batched mean-shift kernels against the float64 reference of tests/ms_f64.py, at the sizes where they branch.

Every case runs through `MeanShiftTorch.fit_segments` in all four modes:
  * the exact outputs (every point's inlier count, max_idx, n_in, labels) are bit-exact;
  * strict / no_freeze: |T - T64| <= 1, T == T64 unless the float64 largest shift at T-1 or T is within 1e-4 of
    the threshold or within ms_f64.shift_tol (the kernels' fp32 shift error bound) of it, and the centre within ms_f64.centre_bound of the float64 star at the kernel's own T;
  * early_exit / certified: the reported iteration count <= T64 + 1 (for certified this is the witness kernel's
    it0, a claimed lower bound of the reference's T) and the centre within delta + bound of the star at T64 --
    the conclusion of the certificate (DESIGN section 5), fit by fit.
Sizes straddle the kernels' edges: the 1024-point density tiles, the pruned density pass and the shared-memory sweep
tiles (4096 points), odd tails; one call holds more fits than a launch chunk (2048).  Each check is also run against
deliberately wrong references, and the tests assert that every one of them is caught.
"""
import numpy as np
import pytest
import torch

import ms_f64
from pvn3d_b200.meanshift import MeanShiftTorch

pytestmark = pytest.mark.gpu
MODES = ["certified", "strict", "no_freeze", "early_exit"]
NS = [1, 2, 3, 255, 257, 1023, 1024, 1025, 2047, 2049, 4095, 4096, 4097, 8193]
KINDS = ["votes", "two", "dups", "clean", "far"]
BWS = [0.02, 0.08, 0.16]
CENTRE = np.array([0.1, -0.05, 0.9])
K_FIT_MAX, K_PT_TILE = 2048, 4096


def make_cloud(kind, n, bw, seed):
    """[n,3] float32 votes of one fit"""
    rng = np.random.default_rng(seed)
    if kind == "votes":            # vote-like: 5 mm noise, 10-30 % outliers in the object's box
        A = CENTRE + rng.normal(0, 0.005, (n, 3))
        k = int(round(rng.uniform(0.1, 0.3) * n))
        A[rng.choice(n, k, replace=False)] = rng.uniform(CENTRE - [0.5, 0.4, 0.3], CENTRE + [0.5, 0.4, 0.3], (k, 3))
    elif kind == "two":            # two clusters of near-equal density, 3 bw apart
        h = n // 2
        A = np.concatenate([CENTRE + rng.normal(0, 0.2 * bw, (h, 3)),
                            CENTRE + [3 * bw, 0, 0] + rng.normal(0, 0.2 * bw, (n - h, 3))])
        A = A[rng.permutation(n)]
    elif kind == "dups":           # exact duplicates: many points share the largest count
        base = CENTRE + rng.normal(0, 0.3 * bw, (max(1, n // 8), 3))
        A = base[rng.integers(0, len(base), n)]
    elif kind == "clean":          # clean cluster: the reference's rule fires before the star is stationary
        A = CENTRE + rng.normal(0, 0.15 * bw, (n, 3))
    elif kind == "far":            # 300 m from the origin
        A = np.array([120.0, -75.0, 300.0]) + rng.normal(0, 0.5 * bw, (n, 3))
        k = n // 5
        A[rng.choice(n, k, replace=False)] += rng.uniform(-0.4, 0.4, (k, 3))
    else:
        raise ValueError(kind)
    return A.astype(np.float32)


# (n, bw, kind, max_iter): every size with two cloud types and bandwidths, plus the iteration caps
CASES = [(n, BWS[(i + j) % 3], KINDS[(2 * i + j) % 5], 300) for i, n in enumerate(NS) for j in range(2)]
CASES += [(1025, 0.08, "votes", 0), (257, 0.08, "votes", 1), (2049, 0.08, "votes", 5), (4097, 0.02, "votes", 5),
          (3, 0.16, "two", 1), (1, 0.08, "clean", 0)]
assert any(n <= K_PT_TILE for n, *_ in CASES) and any(n > K_PT_TILE for n, *_ in CASES)
assert any(n % 2 for n, *_ in CASES) and {1023, 1025, 4095, 4096, 4097} <= {n for n, *_ in CASES}
assert {k for _, _, k, _ in CASES} == set(KINDS) and {b for _, b, _, _ in CASES} == set(BWS)
assert {m for *_, m in CASES} == {0, 1, 5, 300}

WORST = {}


def _note(check, ratio):
    WORST[check] = max(WORST.get(check, 0.0), float(ratio))


def run_fits(clouds, bw, max_iter, mode, dev, brute=False):
    """one fit_segments call over all clouds -> dict of host arrays"""
    counts = [len(c) for c in clouds]
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)
    total = int(sum(counts))
    pts = torch.zeros((max(total, 1), 4), dtype=torch.float32, device=dev)
    if total:
        pts[:total, :3] = torch.from_numpy(np.concatenate([c for c in clouds if len(c)])).to(dev)
    ms = MeanShiftTorch(bw, max_iter=max_iter, mode=mode)
    ms.brute_density = brute
    ctr, labels, mi, n_in = ms.fit_segments(pts, torch.tensor(starts, dtype=torch.int32, device=dev),
                                            torch.tensor(counts, dtype=torch.int32, device=dev))
    return dict(ctr=ctr.cpu().numpy(), labels=labels.cpu().numpy().astype(bool), mi=mi.cpu().numpy(),
                n_in=n_in.cpu().numpy(), counts=ms.last_counts()[:total].cpu().numpy(), starts=starts,
                certified=ms.certified_fits() if mode == "certified" else None)


def check_exact(out, f, n, ref):
    s = out["starts"][f]
    assert np.array_equal(out["counts"][s:s + n], ref["num_in"]), "inlier counts"
    assert int(out["mi"][f]) == ref["max_idx"], (int(out["mi"][f]), ref["max_idx"])
    assert int(out["n_in"][f]) == int(ref["num_in"][ref["max_idx"]])
    assert np.array_equal(out["labels"][s:s + n], ref["labels"]), "labels"


_groups = sorted({(bw, mi) for _, bw, _, mi in CASES})


@pytest.fixture(scope="module")
def refs(cuda_dev):
    out = {}
    for bw, max_iter in _groups:
        cs = [(i, c) for i, c in enumerate(CASES) if c[1] == bw and c[3] == max_iter]
        clouds = [make_cloud(k, n, bw, 100 + i) for i, (n, _, k, _) in cs]
        out[(bw, max_iter)] = ([i for i, _ in cs], clouds, ms_f64.reference(clouds, bw, max_iter, cuda_dev))
    return out


@pytest.fixture(scope="module")
def kernel_runs(cuda_dev, refs):
    return {(g, mode): run_fits(refs[g][1], g[0], g[1], mode, cuda_dev) for g in _groups for mode in MODES}


@pytest.mark.parametrize("mode", MODES)
def test_fits_against_float64(refs, kernel_runs, mode):
    for g in _groups:
        idx, clouds, ref = refs[g]
        out = kernel_runs[(g, mode)]
        bw = g[0]
        for f, (ci, A, r) in enumerate(zip(idx, clouds, ref)):
            check_exact(out, f, len(A), r)
            ok, ratio, msg = ms_f64.check_fit(mode, r, out["ctr"][f, :3], int(out["ctr"][f, 3]), bw)
            _note(f"centre/{mode}", ratio)
            assert ok, (CASES[ci], mode, msg)
            # the stated bound is ten times tighter than the 1e-4 relative parity bar
            assert ms_f64.centre_bound(r["traj"][r["T"]], bw) <= 1e-5 * np.linalg.norm(r["traj"][r["T"]])


def test_certified_runs_take_both_paths(refs, kernel_runs):
    closed = sum(kernel_runs[(g, "certified")]["certified"] for g in _groups)
    nonempty = sum(len(refs[g][1]) for g in _groups)
    assert 0 < closed < nonempty, (closed, nonempty)


def test_wrong_references_are_caught(cuda_dev, refs, kernel_runs):
    """each check fails against a deliberately wrong reference"""
    caught = dict.fromkeys(["T+2", "last_tie", "drop_past_4096", "second_star"], False)
    for g in _groups:
        idx, clouds, ref = refs[g]
        bw, max_iter = g
        strict = kernel_runs[(g, "strict")]
        cert = kernel_runs[(g, "certified")]
        for f, (ci, A, r) in enumerate(zip(idx, clouds, ref)):
            it = int(strict["ctr"][f, 3])
            wrong = dict(r, T=r["T"] + 2, traj=np.concatenate([r["traj"], r["traj"][-1:].repeat(2, 0)]),
                         shifts=np.concatenate([r["shifts"], [0.0, 0.0]]))
            if not ms_f64.check_fit("strict", wrong, strict["ctr"][f, :3], it, bw)[0]:
                caught["T+2"] = True
            last = len(A) - 1 - int(np.argmax(r["num_in"][::-1]))
            if last != r["max_idx"]:
                s = strict["starts"][f]
                lab = np.asarray(torch.norm(torch.from_numpy(A) - torch.from_numpy(A[last]), dim=1) < bw)
                if not np.array_equal(strict["labels"][s:s + len(A)], lab) or int(strict["mi"][f]) != last:
                    caught["last_tie"] = True
            if len(A) > K_PT_TILE:
                cut = ms_f64.exact_part(A[:K_PT_TILE], bw)
                s = strict["starts"][f]
                if not np.array_equal(strict["counts"][s:s + K_PT_TILE], cut[0]):
                    caught["drop_past_4096"] = True
            far = np.linalg.norm(A.astype(np.float64) - A[r["max_idx"]], axis=1) >= 2 * bw
            if far.any() and max_iter == 300:
                j = int(np.flatnonzero(far)[np.argmax(r["num_in"][far])])
                w2 = ms_f64.iterate_f64([A], bw, max_iter, [j], cuda_dev)[0]
                ok = ms_f64.check_fit("certified", w2, cert["ctr"][f, :3], int(cert["ctr"][f, 3]), bw)[0]
                if not ok:
                    caught["second_star"] = True
    assert all(caught.values()), caught


def test_float32_threshold_on_pairs_at_bandwidth(cuda_dev):
    """pairs at bw +- 1e-7: the kernels follow the float32 test sqrt(d2) < float32(bw), not a float64 one"""
    bw = 0.08
    p = np.array([0.1, -0.05, 0.9], np.float32)
    d = np.linspace(bw - 1e-7, bw + 1e-7, 84)
    axes = np.concatenate([np.eye(3), -np.eye(3)])[np.arange(84) % 6]     # ring points of one axis see each other only
    ring = (p + d[:, None] * axes).astype(np.float32)
    A = np.concatenate([np.repeat(p[None], 200, 0), ring]).astype(np.float32)
    ref = ms_f64.exact_part(A, bw)
    assert ref[1] == 0
    wrong = np.linalg.norm(A.astype(np.float64) - A[0].astype(np.float64), axis=1) < bw
    assert not np.array_equal(wrong, ref[2]), "the case must separate the float32 and float64 thresholds"
    for mode in MODES:
        out = run_fits([A], bw, 300, mode, cuda_dev)
        check_exact(out, 0, len(A), dict(num_in=ref[0], max_idx=ref[1], labels=ref[2]))
        assert not np.array_equal(out["labels"][:len(A)], wrong)


CHUNK_WRONG = [2052, 2300, 2598]     # second-chunk fits whose first-chunk partner (f - 2048) has the same size


def _chunk_clouds():
    """2600 fits: small vote sets, empty fits on both sides of index 2048, fits above 4096 points in both chunks"""
    rng = np.random.default_rng(7)
    sizes = rng.integers(5, 160, 2600)
    sizes[[3, 2046, 2047, 2048, 2049, 2599]] = 0
    sizes[[100, 2300]] = [4097, 5000]
    sizes[[2050, 2051]] = [1, 2]
    for f in CHUNK_WRONG:
        sizes[f - K_FIT_MAX] = sizes[f]
    clouds = [make_cloud("votes" if i % 3 else "two", int(n), 0.08, 5000 + i) if n else np.zeros((0, 3), np.float32)
              for i, n in enumerate(sizes)]
    return clouds


def _exact_ok(out, f, n, ref):
    s = out["starts"][f]
    return (np.array_equal(out["counts"][s:s + n], ref["num_in"]) and int(out["mi"][f]) == ref["max_idx"]
            and np.array_equal(out["labels"][s:s + n], ref["labels"]))


@pytest.mark.parametrize("mode", ["certified", "strict"])
def test_chunked_call_equals_standalone_fits(cuda_dev, mode):
    """certified: every fit of the 2600-fit call equals its stand-alone fit bit for bit.  strict: the all-seed sweep
    picks its variant from the launch's total seed count, so shifts may round differently and T move by one; there
    the exact outputs are equal and both centres are within the float64 bound of the float64 star at their own T."""
    clouds = _chunk_clouds()
    assert K_FIT_MAX < len(clouds) <= 4500
    assert any(len(c) > K_PT_TILE for c in clouds[K_FIT_MAX:]) and len(clouds[K_FIT_MAX]) == 0
    assert all(len(clouds[f]) == len(clouds[f - K_FIT_MAX]) > 0 for f in CHUNK_WRONG)
    bw = 0.08
    out = run_fits(clouds, bw, 300, mode, cuda_dev)
    ref = ms_f64.reference(clouds, bw, 300, cuda_dev)
    for f, (A, r) in enumerate(zip(clouds, ref)):
        if len(A) == 0:
            continue
        one = run_fits([A], bw, 300, mode, cuda_dev)
        s = out["starts"][f]
        assert np.array_equal(out["labels"][s:s + len(A)], one["labels"][:len(A)]), f
        assert out["mi"][f] == one["mi"][0] and out["n_in"][f] == one["n_in"][0], f
        check_exact(out, f, len(A), r)
        ok, ratio, msg = ms_f64.check_fit(mode, r, out["ctr"][f, :3], int(out["ctr"][f, 3]), bw)
        _note(f"chunked/{mode}", ratio)
        assert ok, (f, msg)
        if mode == "certified":
            assert np.array_equal(out["ctr"][f], one["ctr"][0]), f
        else:
            ok1, _, msg1 = ms_f64.check_fit(mode, r, one["ctr"][0, :3], int(one["ctr"][0, 3]), bw)
            assert ok1, (f, "stand-alone", msg1)
            tb, ta = int(out["ctr"][f, 3]), int(one["ctr"][0, 3])
            allowed = (ms_f64.centre_bound(r["traj"][tb], bw) + ms_f64.centre_bound(r["traj"][ta], bw)
                       + float(np.linalg.norm(r["traj"][tb] - r["traj"][ta])))
            diff = float(np.linalg.norm(out["ctr"][f, :3].astype(np.float64) - one["ctr"][0, :3]))
            _note("chunked/strict vs stand-alone", diff / allowed)
            assert diff <= allowed, (f, diff, allowed)
    # wrong reference: a second-chunk fit read at the first chunk's offsets (a fit of the same size)
    for f in CHUNK_WRONG:
        r = ref[f - K_FIT_MAX]
        ok = _exact_ok(out, f, len(clouds[f]), r) and \
            ms_f64.check_fit(mode, r, out["ctr"][f, :3], int(out["ctr"][f, 3]), bw)[0]
        assert not ok, f


@pytest.mark.parametrize("n", [1, 2, 3, 255, 257, 1023, 1024, 1025, 2047, 2049, 4095, 4096, 4097])
def test_pruned_density_at_size_edges(cuda_dev, n):
    """the pruned and the brute-force density passes give every point the oracle's exact count at the tile and
    shared-memory edges (fits above 4096 points take the brute-force kernel in both runs)"""
    bw = 0.08
    clouds = [make_cloud("votes", n, bw, n), make_cloud("dups", n, bw, n + 1)]
    refs = [ms_f64.exact_part(A, bw) for A in clouds]
    for brute in (False, True):
        out = run_fits(clouds, bw, 300, "certified", cuda_dev, brute=brute)
        for f, (A, r) in enumerate(zip(clouds, refs)):
            check_exact(out, f, len(A), dict(num_in=r[0], max_idx=r[1], labels=r[2]))


def test_zz_report_worst_ratios():
    """prints the worst |got - ref| / bound of each check of this module (run last)"""
    for k, v in sorted(WORST.items()):
        print(f"F64RATIO {k} {v:.4f}")
