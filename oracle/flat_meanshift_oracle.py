"""NumPy float64 statement of sklearn's flat-kernel MeanShift(bandwidth=bw, bin_seeding=True) as
pvn3d/eval_icp.py:56-64 (`get_cld_bigest_clus`) runs it, and of the filter + ICP pipeline of
pvn3d_b200's clustered refiner -- a checker, written from the documented steps:

1. bin seeds: key = round-half-even(x / bw) per coordinate (float64 division); bins in order of first
   occurrence; seed = float32(key) * float32(bw) in float32.  If every point has its own bin the
   seeds are the points themselves.
2. hill climb per seed: members d2 <= bw*bw with d2 = (dx*dx + dy*dy) + dz*dz; no members -> stop
   (count 0); mean = sequential float64 sum of the members in index order / count; stop when
   sqrt((ddx*ddx + ddy*ddy) + ddz*ddz) <= 1e-3*bw or iteration == max_iter.
   n_iter = max over every seed of its completed iterations.
3. collapse: seeds with count > 0; equal centres (==) are one entry with the FIRST seed's centre
   and the LAST seed's count.
4. order by (count, x, y, z) descending.
5. greedy de-duplication: a kept centre removes every later one with d2 <= bw*bw.
6. labels: nearest kept centre by the same d2, lowest index on ties.

sklearn sums each seed's members in its neighbour search's order, so it agrees with this statement
to rounding (labels and n_iter equal, centres to ~1e-15 on eval_icp-like clouds); the GPU kernel
follows this statement bit for bit.
"""
from __future__ import annotations

import numpy as np

from oracle import icp_oracle


def _d2(P: np.ndarray, c) -> np.ndarray:
    d = P - np.asarray(c, np.float64)
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def bin_seeds(X: np.ndarray, bw: float) -> np.ndarray:
    """step 1: seeds [S,3] (float32 values, or X itself when every point has its own bin)"""
    bins = {}
    for k in np.round(X / bw):
        bins.setdefault(tuple(k), None)
    if len(bins) == len(X):
        return X
    return np.array(list(bins), dtype=np.float32) * np.float32(bw)


def climb(seed, X: np.ndarray, bw: float, max_iter: int):
    """step 2: (centre tuple, member count of the last pass, completed iterations)"""
    bw2, thresh = bw * bw, 1e-3 * bw
    mean = np.asarray(seed, np.float64)
    it = 0
    while True:
        members = X[_d2(X, mean) <= bw2]
        if len(members) == 0:
            break
        old = mean
        mean = np.add.reduce(members, axis=0) / len(members)  # row by row: a sequential sum per column
        dd = mean - old
        if np.sqrt((dd[0] * dd[0] + dd[1] * dd[1]) + dd[2] * dd[2]) <= thresh or it == max_iter:
            break
        it += 1
    return tuple(mean), len(members), it


def flat_mean_shift(X, bw: float, max_iter: int = 300, return_counts: bool = False):
    """-> (cluster_centers [K,3] f64, labels [n] i64, n_iter) and, with return_counts, the member
    count of each kept centre [K].  Raises ValueError when no seed has a member (as sklearn does)."""
    X = np.ascontiguousarray(X, np.float64)
    bw = float(bw)
    res = [climb(s, X, bw, max_iter) for s in bin_seeds(X, bw)]
    n_iter = max(r[2] for r in res)
    entries = {}
    for c, cnt, _ in res:
        if cnt:
            entries[c] = cnt              # a dict keeps the first key and the last value
    if not entries:
        raise ValueError(f"no point within bandwidth={bw} of any seed")
    items = sorted(entries.items(), key=lambda kv: (kv[1], kv[0]), reverse=True)
    centres = np.array([c for c, _ in items], np.float64)
    counts = np.array([n for _, n in items], np.int64)
    keep = np.ones(len(centres), bool)
    for i in range(len(centres)):
        if keep[i]:
            later = _d2(centres[i + 1:], centres[i]) <= bw * bw
            keep[i + 1:] &= ~later
    centres, counts = centres[keep], counts[keep]
    d2 = np.stack([_d2(X, c) for c in centres], 1)
    labels = np.argmin(d2, axis=1)        # first minimum: the lower index on ties
    return (centres, labels, n_iter, counts) if return_counts else (centres, labels, n_iter)


def biggest_cluster(X, bw: float = 0.06, max_iter: int = 300) -> np.ndarray:
    """indices of the points labelled 0 (the kept cluster of eval_icp's get_cld_bigest_clus), ascending"""
    _, labels, _ = flat_mean_shift(X, bw, max_iter)
    return np.nonzero(labels == 0)[0]


def clustered_fit(model, pcld_frame, mask_frame, cls: int, init, max_pts: int, max_iter: int, tol: float,
                  bw: float, cluster_max_iter: int = 300, nn=icp_oracle.nearest):
    """the clustered refiner's fit of one (frame, class): the strided selection, the biggest flat
    mean-shift cluster of it, then my_icp on those points.  Returns (T, distances, i, kept count)."""
    sel = icp_oracle.select(mask_frame, cls, max_pts)
    B = np.asarray(pcld_frame)[sel]
    kept = biggest_cluster(B.astype(np.float64), bw, cluster_max_iter)
    T, d, i = icp_oracle.my_icp(model, B[kept], init, max_iter, tol, nn=nn)
    return T, d, i, len(kept)
