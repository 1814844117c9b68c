"""Flat mean shift on the GPU (csrc/flat_meanshift.cuh): the sklearn goldens, bit-identity with the
NumPy oracle on batches and on edge cases built from dyadic coordinates (so that the ties really occur),
and the clustered ICP refiner against the oracle pipeline."""
import os

import numpy as np
import pytest
import torch

from oracle import flat_meanshift_oracle as fmo
from oracle import icp_oracle
from pvn3d_b200 import synth
from pvn3d_b200.eval_utils import pose_add_adds
from pvn3d_b200.icp import IcpRefiner, get_cld_bigest_clus
from pvn3d_b200.meanshift import flat_mean_shift, flat_mean_shift_batch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flat_ms_cases.npz")
TOL_T = 1e-9
TOL_D = 1e-9
BW = 0.0625      # dyadic: keys, distances and bw*bw are exact on dyadic coordinates


def golden_cases():
    z = np.load(GOLDEN)
    for k, name in enumerate(z["names"]):
        p = f"c{k}_"
        yield (str(name), z[p + "X"], float(z[p + "bw"]), z[p + "centers"], z[p + "labels"], int(z[p + "n_iter"]))


@pytest.mark.parametrize("case", list(golden_cases()), ids=lambda c: c[0])
def test_matches_sklearn_goldens(cuda_dev, case):
    name, X, bw, C, L, it = case
    Cg, Lg, itg = flat_mean_shift(X, bw, device=cuda_dev)
    assert itg == it and np.array_equal(Lg, L)
    assert Cg.shape == C.shape and np.abs(Cg - C).max() <= 1e-12
    kept = get_cld_bigest_clus(X, radius=bw, device=cuda_dev)
    assert kept.dtype == X.dtype and np.array_equal(kept, X[L == 0])


def test_bigest_clus_keeps_input_type_and_dtype(cuda_dev):
    _, X, bw, _, _, _ = next(golden_cases())
    X32 = X.astype(np.float32)
    _, L, _ = flat_mean_shift(X32, bw, device=cuda_dev)           # clustered as float64, like eval_icp's cloud
    got = get_cld_bigest_clus(X32, radius=bw, device=cuda_dev)
    assert got.dtype == np.float32 and np.array_equal(got, X32[L == 0])
    t = torch.from_numpy(X32).to(cuda_dev)
    got_t = get_cld_bigest_clus(t, radius=bw, device=cuda_dev)
    assert torch.is_tensor(got_t) and got_t.dtype == torch.float32 and got_t.device == t.device
    assert np.array_equal(got_t.cpu().numpy(), X32[L == 0])


def run_batch(clouds, bw, max_iter, dev):
    """every cloud in one launch -> per cloud (centres, counts, labels, n_iter)"""
    off = np.concatenate([[0], np.cumsum([len(c) for c in clouds])]).astype(np.int32)
    X = torch.from_numpy(np.concatenate(clouds).astype(np.float64)).to(dev)
    lab, ctr, cnt, ncl, nit = flat_mean_shift_batch(X, off, bw, max_iter)
    lab, ctr, cnt, ncl, nit = (t.cpu().numpy() for t in (lab, ctr, cnt, ncl, nit))
    out = []
    for f in range(len(clouds)):
        a, k = off[f], ncl[f]
        out.append((ctr[a:a + k], cnt[a:a + k], lab[a:off[f + 1]], int(nit[f])))
    return out


def assert_exact(clouds, bw, max_iter, dev):
    for X, (C, N, L, it) in zip(clouds, run_batch(clouds, bw, max_iter, dev)):
        Co, Lo, ito, No = fmo.flat_mean_shift(X, bw, max_iter, return_counts=True)
        assert it == ito
        assert np.array_equal(C, Co) and np.array_equal(N, No) and np.array_equal(L, Lo)


def dyadic(rng, n, span, q=2.0 ** -6):
    return np.round(rng.uniform(-span, span, (n, 3)) / q) * q


def test_bit_identical_to_oracle_on_icp_batch(cuda_dev):
    data = synth.make_icp_batch(16, 5, 2000, seed=31, outlier_frac=0.1, n_stray=200)
    clouds = []
    for b in range(16):
        for c in np.nonzero(data["present"][b])[0]:
            sel = icp_oracle.select(data["mask"][b], c, 2000)
            clouds.append(data["pcld"][b][sel].astype(np.float64))
    assert len(clouds) == 80
    assert_exact(clouds, 0.06, 300, cuda_dev)


def test_keys_at_half_round_to_even(cuda_dev):
    k = np.array([-2.5, -1.5, -0.5, 0.5, 1.5, 2.5, 3.5])
    g = np.stack(np.meshgrid(k, k, k[:3], indexing="ij"), -1).reshape(-1, 3) * BW
    assert np.all(np.round(g / BW) % 2 == 0)                          # every key rounded to an even integer
    assert_exact([g, g[::-1].copy(), g[::3].copy()], BW, 300, cuda_dev)


def test_member_at_exactly_bw(cuda_dev):
    # the seed of the middle bin sits on the middle point; its neighbours lie exactly bw away
    X = np.array([[0.0, 0.0, 0.0], [BW, 0.0, 0.0], [-BW, 0.0, 0.0], [0.0, BW, 0.0], [0.0, 0.0, 0.0]])
    assert np.any(fmo._d2(X, X[0]) == BW * BW)
    assert_exact([X], BW, 300, cuda_dev)
    C, L, _ = fmo.flat_mean_shift(X, BW)
    assert len(C) == 1 and np.all(L == 0)                             # included: one cluster


def test_centre_at_exactly_bw_from_stronger_one_is_removed(cuda_dev):
    # A's four points (keys +-0.5 round to 0) climb to 0, B's two to (bw, 0, 0): neither ball holds the
    # other's points, and the weaker centre lies exactly bw from the stronger one
    e = BW / 2
    A = np.array([[0, e, 0], [0, -e, 0], [0, 0, e], [0, 0, -e]])
    B = np.array([[BW, e, 0], [BW, -e, 0]])
    X = np.concatenate([A, B])
    res = [fmo.climb(s, X, BW, 300) for s in fmo.bin_seeds(X, BW)]
    assert sorted((r[1], r[0]) for r in res) == [(2, (BW, 0.0, 0.0)), (4, (0.0, 0.0, 0.0))]
    C, L, _ = fmo.flat_mean_shift(X, BW)
    assert C.tolist() == [[0.0, 0.0, 0.0]] and np.all(L == 0)
    assert_exact([X, X[::-1].copy()], BW, 300, cuda_dev)


def test_point_equidistant_from_two_centres_takes_lower_index(cuda_dev):
    X = dyadic(np.random.default_rng(0), 60, 0.15, q=2.0 ** -4)
    C, L, _ = fmo.flat_mean_shift(X, BW)
    d2 = np.stack([fmo._d2(X, c) for c in C], 1)
    assert ((d2 == d2.min(1, keepdims=True)).sum(1) > 1).any()       # the tie occurs
    assert_exact([X], BW, 300, cuda_dev)


def test_collapse_keeps_first_centre_and_last_count(cuda_dev):
    # max_iter 0: the seeds of bins (0,0,0) and (1,0,0) both reach (0.625 bw, 0, 0) after one mean, with
    # 4 and 6 members.  The entry keeps the count of the LAST of them: 6 in one row order, 4 (not the
    # larger) when the bins occur the other way round.
    a, b, u = [0.375, 0.0, 0.0], [0.875, 0.0, 0.0], [[0.625, 0.875, 0.0], [0.625, -0.875, 0.0]]
    for rows, want in (([a, b, a, b], 6), ([b, a, b, a], 4)):
        X = np.array(rows + u) * BW
        res = [fmo.climb(s, X, BW, 0) for s in fmo.bin_seeds(X, BW)]
        same = [r[1] for r in res if r[0] == (0.625 * BW, 0.0, 0.0)]
        assert len(same) == 2 and same[0] != same[1] and same[1] == want   # distinct counts collapse
        C, _, _, N = fmo.flat_mean_shift(X, BW, 0, return_counts=True)
        assert C.tolist() == [[0.625 * BW, 0.0, 0.0]] and N.tolist() == [want]
        assert_exact([X], BW, 0, cuda_dev)


def test_seeds_converging_to_one_centre(cuda_dev):
    # bins split a tight blob: several seeds climb to the same mean and collapse into one entry
    rng = np.random.default_rng(3)
    X = np.round((rng.normal(0.0, 0.02, (400, 3)) + BW / 2) / 2.0 ** -8) * 2.0 ** -8
    res = [fmo.climb(s, X, BW, 300) for s in fmo.bin_seeds(X, BW)]
    centres = [r[0] for r in res if r[1]]
    assert len(set(centres)) < len(centres)                           # a collapse happens
    assert_exact([X], BW, 300, cuda_dev)


def test_fallback_max_iter_and_tiny_fits(cuda_dev):
    rng = np.random.default_rng(4)
    sparse = np.arange(64)[:, None] * np.array([[3 * BW, 0.0, 0.0]]) + [0.0, 0.01, 0.0]
    assert len(fmo.bin_seeds(sparse, BW)) == len(sparse)
    assert_exact([sparse, np.array([[0.1, 0.2, 0.3]]), np.array([[0.1, 0.2, 0.3], [0.13, 0.2, 0.3]])], BW, 300,
                 cuda_dev)
    _, X, bw, _, _, it = next(c for c in golden_cases() if c[0] == "large_split")
    for m in (0, 1, 2, it // 2):                                      # max_iter reached
        assert_exact([X], bw, m, cuda_dev)
    assert_exact([dyadic(rng, 3000, 0.3)], BW, 300, cuda_dev)


def test_mixed_batch_of_1_to_4096_points(cuda_dev):
    rng = np.random.default_rng(5)
    sizes = [1, 2, 3, 10, 100, 777, 2000, 4096, 5, 4095]
    clouds = [dyadic(rng, n, 0.2) if i % 2 else rng.normal(0, 0.05, (n, 3)) for i, n in enumerate(sizes)]
    assert_exact(clouds, BW, 300, cuda_dev)
    first = run_batch(clouds, BW, 300, cuda_dev)
    again = run_batch(clouds, BW, 300, cuda_dev)
    X = torch.zeros((4097, 3), dtype=torch.float64, device=cuda_dev)
    with pytest.raises(ValueError, match="at most"):                 # the bound comes from the offsets
        flat_mean_shift_batch(X, [0, 4097], BW)
    with pytest.raises(ValueError, match="non-decreasing"):
        flat_mean_shift_batch(X, [0, 9, 5], BW)
    for a, b in zip(first, again):
        assert all(np.array_equal(x, y) for x, y in zip(a, b))


# ---- the clustered refiner ------------------------------------------------------------------------
def _kd_nearest(q, pts, k=4):
    from scipy.spatial import cKDTree
    k = min(k, len(pts))
    _, cand = cKDTree(pts).query(q, k=k)
    cand = cand.reshape(len(q), k)
    d2 = ((q[:, None, :] - pts[cand]) ** 2).sum(-1)
    best = d2.min(1, keepdims=True)
    idx = np.where(d2 == best, cand, np.iinfo(np.int64).max).min(1)
    return np.sqrt(best[:, 0]), idx


@pytest.fixture(scope="module")
def stray_batch():
    return synth.make_icp_batch(16, 5, 2000, seed=13, outlier_frac=0.10, n_stray=200)


def _tensors(data, dev):
    return [torch.from_numpy(np.ascontiguousarray(data[k])).to(dev) for k in ("pcld", "mask", "init", "present")]


def _refiner(data, dev, **kw):
    b, n, _ = data["pcld"].shape
    return IcpRefiner(data["models"], len(data["models"]), b, n, device=dev, **kw)


def test_clustered_refiner_matches_oracle_pipeline(cuda_dev, stray_batch):
    data = stray_batch
    ref = _refiner(data, cuda_dev, max_pts=2000, min_pts=1500, cluster_bandwidth=0.06)
    out = [o.cpu().numpy() for o in ref.refine(*_tensors(data, cuda_dev))]
    poses, iters, err, refined = out
    kept = ref.cluster_pts.cpu().numpy()
    lists = ref.kept_points().cpu().numpy()
    n_fit = 0
    for b in range(16):
        for c in range(ref.n_cls):
            if not data["present"][b, c]:
                assert refined[b, c] == 0 and kept[b, c] == 0
                continue
            init = np.eye(4)
            init[:3] = data["init"][b, c].astype(np.float64)
            T, d, i, nk = fmo.clustered_fit(data["models"][c], data["pcld"][b], data["mask"][b], c, init, 2000, 500,
                                            1e-9, 0.06, nn=_kd_nearest)
            assert refined[b, c] == 1 and kept[b, c] == nk
            # the kernel's kept list, frame indices of the strided selection (2200 points > max_pts)
            sel = icp_oracle.select(data["mask"][b], c, 2000)
            assert (data["mask"][b] == c).sum() > 2000
            want = sel[fmo.biggest_cluster(data["pcld"][b][sel].astype(np.float64), 0.06)]
            start = int(((data["mask"][b] >= 1) & (data["mask"][b] < c)).sum())
            assert np.array_equal(lists[b, start:start + nk], want)
            assert iters[b, c] == i, (b, c, iters[b, c], i)
            assert np.abs(poses[b, c] - T[:3]).max() <= TOL_T
            assert abs(err[b, c] - d.mean()) <= TOL_D
            n_fit += 1
    assert n_fit == 80


def test_clustered_refiner_lowers_add_and_is_deterministic(cuda_dev, stray_batch):
    data = stray_batch
    t = _tensors(data, cuda_dev)
    plain = [o.cpu().numpy() for o in _refiner(data, cuda_dev, max_pts=2000, min_pts=1500).refine(*t)]
    ref = _refiner(data, cuda_dev, max_pts=2000, min_pts=1500, cluster_bandwidth=0.06)
    first = [o.cpu().numpy() for o in ref.refine(*t)] + [ref.cluster_pts.cpu().numpy()]
    again = [o.cpu().numpy() for o in ref.refine(*t)] + [ref.cluster_pts.cpu().numpy()]
    for a, b in zip(first, again):
        assert np.array_equal(a, b)
    torch.cuda.synchronize()
    s = torch.cuda.Stream(cuda_dev)
    s.wait_stream(torch.cuda.current_stream(cuda_dev))
    with torch.cuda.stream(s):
        ref.poses.fill_(float("nan"))
        ref.cluster_pts.fill_(-1)
        side = list(ref.refine(*t)) + [ref.cluster_pts]
        done = torch.cuda.Event()
        done.record(s)
    done.synchronize()
    for a, b in zip(first, side):
        assert np.array_equal(a, b.cpu().numpy())
    add_plain, add_filt = [], []
    for b in range(16):
        for c in np.nonzero(data["present"][b])[0]:
            mdl = torch.from_numpy(data["models"][c]).to(cuda_dev)
            gt = torch.from_numpy(data["gt"][b, c]).to(cuda_dev)
            for res, acc in ((plain, add_plain), (first, add_filt)):
                acc.append(float(pose_add_adds(torch.from_numpy(res[0][b, c]).to(cuda_dev), gt, mdl)[0][0]))
    assert np.mean(add_filt) < np.mean(add_plain), (np.mean(add_filt), np.mean(add_plain))


def test_clustered_refine_makes_no_host_sync(cuda_dev):
    data = synth.make_icp_batch(2, 3, 400, seed=4, n_bg=200, n_stray=60)
    ref = _refiner(data, cuda_dev, max_pts=300, min_pts=100, cluster_bandwidth=0.06)
    t = _tensors(data, cuda_dev)
    ref.refine(*t)                                                    # warm
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        ref.refine(*t)
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    torch.cuda.synchronize()


def test_default_refiner_is_unchanged_by_the_option(cuda_dev):
    data = synth.make_icp_batch(4, 5, 1200, seed=8, outlier_frac=0.1)
    t = _tensors(data, cuda_dev)
    a = [o.clone() for o in _refiner(data, cuda_dev, max_pts=1000, min_pts=500).refine(*t)]
    r = _refiner(data, cuda_dev, max_pts=1000, min_pts=500, cluster_bandwidth=None)
    b = r.refine(*t)
    assert r.cluster_pts is None
    for x, y in zip(a, b):
        assert torch.equal(x, y)
