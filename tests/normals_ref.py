"""numpy/scipy float64 restatement of the three contracts of csrc/normals.cu (include/pvn3d_b200.h:
pvn3d_frame_sample, pvn3d_knn_normals): the seeded sampling key and rule, the exact 50-nearest-neighbour set,
and the normal of its covariance.  Test infrastructure: nothing under pvn3d_b200/ imports it.  Nothing here
needs a GPU."""
import numpy as np
from scipy.spatial import cKDTree

K = 50
MIN_VALID = 400
_U64 = np.uint64


def mix64(z):
    """the splitmix64 finaliser on uint64 arrays (wrapping arithmetic)"""
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> _U64(30))) * _U64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> _U64(27))) * _U64(0x94D049BB133111EB)
        return z ^ (z >> _U64(31))


def mix64_int(z: int) -> int:
    """the same finaliser on a Python int, for checking the array form"""
    m = (1 << 64) - 1
    z &= m
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & m
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & m
    return z ^ (z >> 31)


def sample_keys(seed: int, b: int, hw: int):
    """key(seed, b, p) for p in [0, hw): mix(mix(seed + (b + 1) * 0x9E3779B97F4A7C15) + p)"""
    with np.errstate(over="ignore"):
        base = mix64(_U64(seed) + _U64(b + 1) * _U64(0x9E3779B97F4A7C15))
        return mix64(base + np.arange(hw, dtype=np.uint64))


def sample_frame(valid, n: int, seed: int, b: int):
    """(choose [n] int64, ok) of frame b: valid [hw] bool.  n_v > n: the n valid pixels with the smallest keys
    (lowest pixel first on equal keys), ascending; 400 <= n_v <= n: the valid pixels wrapped to n; else zeros."""
    valid = np.asarray(valid, bool).ravel()
    idx = np.nonzero(valid)[0]
    nv = len(idx)
    if nv < MIN_VALID:
        return np.zeros(n, np.int64), 0
    if nv > n:
        keys = sample_keys(seed, b, len(valid))[idx]
        keep = np.lexsort((idx, keys))[:n]
        return np.sort(idx[keep]).astype(np.int64), 1
    return np.pad(idx, (0, n - nv), "wrap").astype(np.int64), 1


def sqdist(q, p):
    """(dx*dx + dy*dy) + dz*dz in float64 of float32 coordinates: q [...,3], p [...,3] broadcast"""
    d = np.asarray(q, np.float32).astype(np.float64) - np.asarray(p, np.float32).astype(np.float64)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _usable(ref, valid):
    ref = np.asarray(ref, np.float32)
    ok = np.isfinite(ref).all(1)
    if valid is not None:
        ok &= np.asarray(valid, bool)
    return np.nonzero(ok)[0]


def knn(ref, query, valid=None, k: int = K):
    """[Q,k] int64 reference indices: the k smallest sqdist, lowest index first on exact ties (-1 rows when
    fewer than k usable points or a non-finite query).  cKDTree finds the k-th distance; every point within
    a slightly larger radius is then re-ranked by the contract's distance and index."""
    ref = np.asarray(ref, np.float32)
    query = np.asarray(query, np.float32)
    use = _usable(ref, valid)
    out = np.full((len(query), k), -1, np.int64)
    if len(use) < k:
        return out
    pts = ref[use].astype(np.float64)
    tree = cKDTree(pts)
    fin = np.isfinite(query).all(1)
    qf = query[fin].astype(np.float64)
    dk, _ = tree.query(qf, k=k)
    r = dk[:, -1] * (1 + 1e-9) + 1e-12
    cands = tree.query_ball_point(qf, r)
    rows = np.nonzero(fin)[0]
    for row, q, c in zip(rows, query[fin], cands):
        ci = use[np.asarray(c, np.int64)]
        d2 = sqdist(q[None], ref[ci])
        order = np.lexsort((ci, d2))[:k]
        out[row] = ci[order]
    return out


def knn_brute(ref, query, valid=None, k: int = K):
    """the same set by a full distance matrix (small clouds only)"""
    ref = np.asarray(ref, np.float32)
    use = _usable(ref, valid)
    out = np.full((len(query), k), -1, np.int64)
    if len(use) < k:
        return out
    for row, q in enumerate(np.asarray(query, np.float32)):
        if not np.isfinite(q).all():
            continue
        d2 = sqdist(q[None], ref[use])
        out[row] = use[np.lexsort((use, d2))[:k]]
    return out


def covariance(ref, idx):
    """C [Q,3,3] float64 = (1/k) sum (p - mean)(p - mean)^T over ref[idx[q]], two passes"""
    p = np.asarray(ref, np.float32)[idx].astype(np.float64)
    c = p - p.mean(1, keepdims=True)
    return np.einsum("qki,qkj->qij", c, c) / idx.shape[1]


def normals(ref, idx, query):
    """(n [Q,3], C [Q,3,3], lam [Q,3] ascending, curvature [Q]) in float64: n = the unit eigenvector of the
    smallest eigenvalue, negated where n . q > 0; zero (and curvature 0) where trace(C) == 0 or idx has -1"""
    q = len(idx)
    n = np.zeros((q, 3))
    C = np.zeros((q, 3, 3))
    lam = np.zeros((q, 3))
    curv = np.zeros(q)
    have = (idx >= 0).all(1)
    if not have.any():
        return n, C, lam, curv
    C[have] = covariance(ref, idx[have])
    w, v = np.linalg.eigh(C[have])
    lam[have] = w
    nn = v[:, :, 0]
    tr = np.trace(C[have], axis1=1, axis2=2)
    qq = np.asarray(query, np.float32)[have].astype(np.float64)
    flip = (nn * qq).sum(1) > 0
    nn[flip] *= -1
    nn[tr == 0] = 0
    n[have] = nn
    curv[have] = np.where(tr > 0, np.maximum(w[:, 0], 0) / np.where(tr > 0, tr, 1), 0)
    return n, C, lam, curv


def frame_input(cloud, valid, rgb, n: int, seed: int, mode: str = "full"):
    """one batch of the builder's outputs from back-projected frames: cloud [B,hw,3] f32, valid [B,hw],
    rgb [B,3,hw] -> dict(choose [B,N] i64, ok [B], cld6 [B,N,6] f32, idx [B,N,50] i64, n [B,N,3] f64, C, lam)"""
    bsz, hw = valid.shape
    out = {k: [] for k in ("choose", "ok", "cld6", "idx", "n", "C", "lam")}
    for b in range(bsz):
        ch, ok = sample_frame(valid[b], n, seed, b)
        out["choose"].append(ch)
        out["ok"].append(ok)
        if not ok:
            out["cld6"].append(np.zeros((n, 6), np.float32))
            out["idx"].append(np.full((n, K), -1, np.int64))
            for k, s in (("n", (n, 3)), ("C", (n, 3, 3)), ("lam", (n, 3))):
                out[k].append(np.zeros(s))
            continue
        pc = cloud[b][ch]
        out["cld6"].append(np.concatenate([pc, rgb[b][:, ch].T.astype(np.float32)], 1))
        if mode == "full":
            idx = knn(cloud[b], pc, valid[b])
            ref = cloud[b]
        else:
            idx = knn(pc, pc)
            ref = pc
        nrm, C, lam, _ = normals(ref, idx, pc)
        out["idx"].append(idx)
        out["n"].append(nrm)
        out["C"].append(C)
        out["lam"].append(lam)
    return {k: np.stack(v) for k, v in out.items()}
