"""Golden vectors of flat-kernel mean shift recorded from sklearn itself (build container only).

Runs `sklearn.cluster.MeanShift(bandwidth=bw, bin_seeding=True).fit(X)` exactly as pvn3d/eval_icp.py's
get_cld_bigest_clus calls it (float64 input, default min_bin_freq=1, cluster_all=True, max_iter=300)
and records X, bw -> (cluster_centers_, labels_, n_iter_) for the cases below into flat_ms_cases.npz.
While recording, it asserts that oracle/flat_meanshift_oracle.py agrees with sklearn: the same labels
and n_iter, centres within 1e-12.  The tests read only the npz.

    python tests/golden/make_golden_flat_ms.py      # writes flat_ms_cases.npz + make_golden_flat_ms.log
"""
import os
import sys
import time
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import flat_meanshift_oracle  # noqa: E402
from pvn3d_b200 import synth  # noqa: E402


def object_cloud(rng, extents, n, outlier_frac=0.0, n_stray=0, stray_dist=0.2):
    """eval_icp-like masked scene points: the visible faces of a box, outliers in its bounding box,
    and a stray blob (a fragment of something else carrying the object's label)"""
    R = synth._haar_rotation(rng)
    t = np.array([0.05, -0.03, 0.8])
    p = synth.visible_box_points(extents, R, t, n, 0.001, rng)
    k = int(round(outlier_frac * n))
    if k:
        p[rng.choice(n, k, replace=False)] = rng.uniform(p.min(0), p.max(0), size=(k, 3))
    if n_stray:
        d = rng.normal(size=3)
        c = t + d / np.linalg.norm(d) * (0.5 * np.linalg.norm(extents) + stray_dist)
        p = np.concatenate([p, c + rng.normal(0.0, 0.005, (n_stray, 3))])
        p = p[rng.permutation(len(p))]
    return p.astype(np.float32).astype(np.float64)    # eval_icp's cloud: float32 depth maths, then float64


def cases():
    rng = np.random.default_rng(2027)
    out = [
        ("eval_icp_regime", object_cloud(rng, (0.10, 0.06, 0.04), 1800, 0.10, n_stray=200), 0.06),
        ("compact_one_cluster", object_cloud(rng, (0.05, 0.04, 0.03), 1500), 0.06),
        ("large_split", object_cloud(rng, (0.30, 0.20, 0.10), 2000, 0.05), 0.06),
    ]
    # two blobs of 300 points with the same spread: equal counts, the order is decided by the centre
    blob = rng.normal(0.0, 0.004, (300, 3))
    two = np.concatenate([blob + [0.1, 0.2, 0.7], blob + [-0.2, 0.2, 0.7]])
    out.append(("equal_count_blobs", two[rng.permutation(len(two))], 0.06))
    # sparse: every point alone in its bin -> the seeds are the points themselves
    sparse = (rng.permutation(np.arange(8 * 8 * 8))[:300, None] // np.array([64, 8, 1]) % 8) * 0.2
    out.append(("sparse_seeds_are_points", sparse + rng.uniform(-0.02, 0.02, sparse.shape), 0.06))
    out.append(("ten_points", rng.uniform(0.0, 0.15, (10, 3)), 0.06))
    out.append(("cap_4096", object_cloud(rng, (0.12, 0.08, 0.05), 3896, 0.10, n_stray=200), 0.06))
    out.append(("bandwidth_0.03", object_cloud(rng, (0.10, 0.06, 0.04), 2000, 0.10, n_stray=150), 0.03))
    return out


def main():
    import sklearn
    from sklearn.cluster import MeanShift

    log = ["make_golden_flat_ms.py: sklearn.cluster.MeanShift(bandwidth, bin_seeding=True).fit(X), X float64",
           f"sklearn {sklearn.__version__}, numpy {np.__version__}"]
    rec, names = {}, []
    for k, (name, X, bw) in enumerate(cases()):
        t0 = time.time()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")            # sklearn warns when the seeds fall back to X
            ms = MeanShift(bandwidth=bw, bin_seeding=True).fit(X)
        dt = time.time() - t0
        C, L, it = ms.cluster_centers_, ms.labels_, ms.n_iter_
        Co, Lo, ito = flat_meanshift_oracle.flat_mean_shift(X, bw)
        seeds = len(flat_meanshift_oracle.bin_seeds(X, bw))
        assert np.array_equal(Lo, L) and ito == it and Co.shape == C.shape, (name, ito, it)
        eC = float(np.abs(Co - C).max())
        assert eC <= 1e-12, (name, eC)
        p = f"c{k}_"
        rec[p + "X"], rec[p + "bw"] = X, np.array(bw)
        rec[p + "centers"], rec[p + "labels"], rec[p + "n_iter"] = C, L.astype(np.int32), np.array(it)
        names.append(name)
        log.append(f"  case {k} {name}: {len(X)} pts, bw {bw:g}, {seeds} seeds -> {len(C)} clusters, "
                   f"n_iter {it}, biggest {int((L == 0).sum())} pts ({dt:.2f}s); "
                   f"oracle: same labels and n_iter, |dC|={eC:.1e}")
        print(log[-1], flush=True)
    rec["names"] = np.array(names)
    path = os.path.join(HERE, "flat_ms_cases.npz")
    np.savez_compressed(path, **rec)
    log.append(f"wrote {os.path.basename(path)} ({os.path.getsize(path)} bytes): oracle == sklearn on every case")
    print(log[-1])
    with open(os.path.join(HERE, "make_golden_flat_ms.log"), "w") as f:
        f.write("\n".join(log) + "\n")


if __name__ == "__main__":
    main()
