"""References, cloud builders and wrong references ("mutants") for the checks of the coordinate-only kernels of hot
path A: furthest-point sampling, ball query, 3-NN, the inverse-distance weights, the SA factor table and centre term.

The index ops have a literal reference already (oracle/pn2_oracle.c); what is here is
  * numpy restatements of the three small value kernels (weights_ref is float32 operation by operation, so the check
    is bit-exact; weights_f64 / centre_term_f64 are the mathematical operation in float64 with a stated bound),
  * seeded clouds built to hit what goes wrong in such kernels: exact ties, coincident points, tight boxes, points
    within an ulp of a radius, far and tiny coordinate scales,
  * mutants: each takes correct oracle output (or the same input) and returns what a plausible kernel mistake would
    give.  A test asserts `kernel == reference` AND `reference != mutant` on the same input, so an input that cannot
    tell the two apart fails the test instead of silently proving nothing.
Nothing here needs a GPU.
"""
import numpy as np

from oracle import pn2

F32 = np.float32
EPS = F32(1e-8)                      # the kernel's 1e-8f (pointnet2_modules.py:184 adds 1e-8 to a float32 tensor)


def bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def same_bits(a, b):
    """float arrays equal bit for bit where finite or inf, NaN exactly where the other is NaN (NaN payloads differ
    between the GPU and the host's divider and carry no information)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(bits(a)[~na], bits(b)[~nb])


# ---- inverse-distance weights ----------------------------------------------------------------------------------
def weights_ref(d2):
    """nn_weights_kernel operation by operation in float32: r_t = 1 / (sqrt(d2_t) + 1e-8f), w_t = r_t / ((r1 + r2) + r3).
    d2 = 0 gives r = 1e8 (a query ON a known point: every level-i point is also a level-(i-1) point), d2 = inf gives
    r = 0 and weight exactly 0 (fewer than three known points), a row of three inf gives 0 / 0 = NaN, as torch does."""
    d2 = np.asarray(d2, np.float32)
    with np.errstate(all="ignore"):
        r = F32(1) / (np.sqrt(d2) + EPS)
        norm = (r[..., 0] + r[..., 1]) + r[..., 2]
        w = r / norm[..., None]
    assert w.dtype == np.float32
    return w


def weights_f64(d2):
    """the same expression (pointnet2_modules.py:183-186) in float64 from the float32 d2"""
    d = np.asarray(d2, np.float32).astype(np.float64)
    with np.errstate(all="ignore"):
        r = 1.0 / (np.sqrt(d) + np.float64(EPS))
        return r / r.sum(-1, keepdims=True)


#: |weights_ref - weights_f64| <= WEIGHTS_ULPS * 2^-24 * |weights_f64|: sqrt, add, divide (1.5 ulp on r), two adds
#: on the norm, one divide -- under 5 half-ulps; 8 leaves room and is still far below any wrong formula
WEIGHTS_ULPS = 8.0


def weights_err_over_bound(w32, w64):
    w32 = np.asarray(w32, np.float64)
    ok = np.isfinite(w64)
    assert np.array_equal(np.isnan(w32), np.isnan(w64))
    bound = WEIGHTS_ULPS * 2.0 ** -24 * np.abs(w64[ok]) + 1e-45
    return float((np.abs(w32[ok] - w64[ok]) / bound).max()) if ok.any() else 0.0


def mut_weights_no_eps(d2):
    d2 = np.asarray(d2, np.float32)
    with np.errstate(all="ignore"):
        r = F32(1) / np.sqrt(d2)
        return r / ((r[..., 0] + r[..., 1]) + r[..., 2])[..., None]


# ---- SA factor table and centre term ---------------------------------------------------------------------------
def tf32(x):
    """cvt.rna.tf32.f32 on finite values: round to nearest, ties away from zero, to 10 mantissa bits"""
    u = bits(x)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def factor_table_ref(xyz, feat, c_feat, k_pad):
    """xyz [R,3], feat [R,ldf] (ldf >= c_feat) or None -> [R,k_pad]: row j = [tf32(f_j) | hi | lo | 0 ..] with
    hi = tf32(x), lo = tf32(x - hi).  x - hi is exact in float32 (hi keeps the leading 11 bits of x)."""
    xyz = np.asarray(xyz, np.float32)
    out = np.zeros((xyz.shape[0], k_pad), np.float32)
    if c_feat:
        out[:, :c_feat] = tf32(np.asarray(feat, np.float32)[:, :c_feat])
    hi = tf32(xyz)
    out[:, c_feat:c_feat + 3] = hi
    out[:, c_feat + 3:c_feat + 6] = tf32(xyz - hi)
    return out


def mut_table_no_lo(table, c_feat):
    out = table.copy()
    out[:, c_feat + 3:c_feat + 6] = 0
    return out


def split_rel_err(xyz, table, c_feat):
    """max |hi + lo - x| / |x| over the non-zero coordinates"""
    x = np.asarray(xyz, np.float64)
    s = table[:, c_feat:c_feat + 3].astype(np.float64) + table[:, c_feat + 3:c_feat + 6].astype(np.float64)
    nz = x != 0
    return float((np.abs(s - x)[nz] / np.abs(x)[nz]).max())


def centre_term_f64(centres, wx, bias):
    """V = c . Wx^T - b in float64 and the bound the fp32 fma chain is held to: 1e-6 (|c| . |Wx|^T + |b|)"""
    c, w, b = (np.asarray(a, np.float64) for a in (centres, wx, bias))
    return c @ w.T - b, 1e-6 * (np.abs(c) @ np.abs(w).T + np.abs(b))


# ---- clouds ([B,n,3] float32, seeded) --------------------------------------------------------------------------
def raster_cloud(b, n, seed, shape="ycb"):
    """what the benchmark feeds: back-projected depth pixels in raster order (synth.make_frame)"""
    from pvn3d_b200 import synth

    return np.stack([synth.make_frame(shape, n_points=n, seed=seed + i).pcld for i in range(b)]).astype(np.float32)


def uniform_cloud(b, n, seed, lo=0.2, hi=1.0):
    return np.random.default_rng(seed).uniform(lo, hi, size=(b, n, 3)).astype(np.float32)


def sorted_cloud(x, axis):
    order = np.argsort(x[..., axis], axis=1, kind="stable")
    return np.take_along_axis(x, order[..., None].repeat(3, -1), 1)


def shuffled(x, seed):
    rng = np.random.default_rng(seed)
    return np.stack([f[rng.permutation(f.shape[0])] for f in x])


def lattice(b, n, step, seed, lo=-20, hi=20, offset=0.0):
    """integer grid points times `step` (+ offset): many exactly equal squared distances"""
    g = np.random.default_rng(seed).integers(lo, hi, size=(b, n, 3)).astype(np.float32)
    return (g * F32(step) + F32(offset)).astype(np.float32)


def with_duplicates(x, seed, groups=None, copies=3):
    """`groups` points per frame are each copied over `copies` other random positions: >= copies + 1 coincident points"""
    rng = np.random.default_rng(seed)
    x = x.copy()
    n = x.shape[1]
    if n < copies + 1:
        return x
    groups = max(1, n // (4 * (copies + 1))) if groups is None else groups
    for f in x:
        perm = rng.permutation(n)[:groups * (copies + 1)].reshape(groups, copies + 1)
        for c in range(1, copies + 1):
            f[perm[:, c]] = f[perm[:, 0]]
    return x


def far(x, offset=300.0):
    return (x + F32(offset)).astype(np.float32)


def tiny(x, scale=1e-4):
    return (x * F32(scale)).astype(np.float32)


def step_ulps(v, k):
    v = F32(v)
    for _ in range(abs(k)):
        v = np.nextafter(v, F32(np.inf if k > 0 else -np.inf), dtype=np.float32)
    return v


SHELL_KS = (0, 1, -1, 2, -2, 8, -8)


def radius_shell(n, m, radii, seed, n_shell_centres=6):
    """One frame built so that `d2 < r2` is decided in the last bits, on a cloud whose 128-point boxes really prune.

    Every centre has x = 0 exactly, y and z on a coarse grid, so a point (+-r_k, y_c, z_c) is at squared distance
    fl(r_k * r_k) from it with no other rounding; r_k = r stepped k float32 ulps, k in SHELL_KS, both signs of x, for
    every radius in `radii` around the first `n_shell_centres` centres.  k = 0 lands ON r2 (strict '<' must reject it),
    the others fall within a few ulps on either side.  The rest of the cloud is uniform in a slab around the centres and
    the whole cloud is sorted by x: a 128-point box is ~1/100 of the slab wide in x, and the sort is arranged so that a
    box STARTS on the innermost shell point of the largest radius (its box distance to the centres' box is that
    point's own squared distance, a few ulps under r2: the block must not be skipped).
    Returns (cloud [1,n,3], centres [1,m,3], shell centre indices)."""
    rng = np.random.default_rng(seed)
    cy = (rng.integers(0, 64, size=m) * F32(1 / 256)).astype(np.float32)              # [0, 0.25), exact
    cz = (F32(0.5) + rng.integers(0, 64, size=m) * F32(1 / 256)).astype(np.float32)
    centres = np.stack([np.zeros(m, np.float32), cy, cz], 1)
    centres[:n_shell_centres, 1] = np.arange(n_shell_centres, dtype=np.float32) * F32(1 / 32) + F32(1 / 512)   # distinct
    shell = []
    for j in range(n_shell_centres):
        for r in radii:
            for k in SHELL_KS:
                rk = step_ulps(r, k)
                for s in (-1, 1):
                    shell.append((F32(s) * rk, centres[j, 1], centres[j, 2]))
    shell = np.array(shell, np.float32)
    rmax = F32(max(radii))
    inner = step_ulps(rmax, min(SHELL_KS))                                              # innermost +x shell point
    nfill = n - len(shell)
    fill = np.stack([rng.uniform(-0.5, 0.5, nfill), rng.uniform(-0.05, 0.3, nfill), rng.uniform(0.45, 0.8, nfill)], 1)
    fill = fill.astype(np.float32)
    fill = fill[np.abs(np.abs(fill[:, 0]) - rmax) > 1e-4]                               # keep the shell's x to itself
    pts = np.concatenate([shell, fill])
    pts = pts[np.argsort(pts[:, 0], kind="stable")]
    first = int(np.searchsorted(pts[:, 0], inner, side="left"))                          # index of the innermost point
    drop = first % 128                                                                  # make it start a 128-box
    keep = np.ones(len(pts), bool)
    keep[np.flatnonzero(pts[:first, 0] < -0.4)[:drop]] = False                          # (far from every centre)
    pts = pts[keep]
    assert len(pts) <= n
    pad = np.repeat(pts[-1:], n - len(pts), 0)                                          # copies of the last (largest x)
    pts = np.concatenate([pts, pad])
    assert int(np.searchsorted(pts[:, 0], inner, side="left")) % 128 == 0
    return pts[None].copy(), centres[None].copy(), np.arange(n_shell_centres)


# ---- mutants of the index ops ----------------------------------------------------------------------------------
def mut_frame0(ref):
    """every frame answers with frame 0's result (a dropped batch offset)"""
    return np.broadcast_to(ref[:1], ref.shape).copy()


def _coincident_last(known):
    """per frame: index -> the highest index holding the same coordinates"""
    out = np.empty(known.shape[:2], np.int32)
    for f, k in enumerate(known):
        _, inv = np.unique(bits(k), axis=0, return_inverse=True)
        inv = inv.reshape(-1)
        last = np.zeros(inv.max() + 1, np.int64)
        np.maximum.at(last, inv, np.arange(len(inv)))
        out[f] = last[inv]
    return out


def mut_nn_last_index(idx, d2, known):
    """3-NN keeping the HIGHEST index among coincident known points instead of the lowest"""
    last = _coincident_last(known)
    out = np.take_along_axis(last, idx.reshape(idx.shape[0], -1).astype(np.int64), 1).reshape(idx.shape)
    out[np.isinf(d2)] = 0
    return out.astype(np.int32)


def mut_nn_ties_unordered(idx, d2):
    """3-NN sorted by distance only: slots of equal distance come out in the other order"""
    out = idx.copy()
    e01, e12 = d2[..., 0] == d2[..., 1], d2[..., 1] == d2[..., 2]
    fin = np.isfinite(d2)
    a = e01 & ~e12 & fin[..., 1]
    out[a, 0], out[a, 1] = idx[a, 1], idx[a, 0]
    b = e12 & ~e01 & fin[..., 2]
    out[b, 1], out[b, 2] = idx[b, 2], idx[b, 1]
    c = e01 & e12 & fin[..., 2]
    out[c, 0], out[c, 2] = idx[c, 2], idx[c, 0]
    return out


def ball_rows_np(centres, cloud, radius, ns, le=False, pad_zero=False):
    """ball query of a few centres of ONE frame restated in numpy on the oracle's squared distances"""
    d2 = pn2.sqdist(centres, cloud)
    r2 = F32(radius) * F32(radius)
    out = np.zeros((len(centres), ns), np.int32)
    for j, row in enumerate(d2):
        hits = np.flatnonzero(row <= r2 if le else row < r2)[:ns]
        if len(hits):
            out[j] = 0 if pad_zero else hits[0]
            out[j, :len(hits)] = hits
    return out


def mut_ball_le(ref, centres, cloud, radius, rows):
    """`d2 <= r2` instead of `d2 < r2`, on the centres `rows` of frame 0"""
    out = ref.copy()
    out[0, rows] = ball_rows_np(centres[0, rows], cloud[0], radius, ref.shape[2], le=True)
    return out


def mut_ball_pad_zero(ref):
    """unfilled slots left 0 instead of repeating the first hit (real hits after slot 0 are larger than it)"""
    out = ref.copy()
    pad = ref[..., 1:] == ref[..., :1]
    out[..., 1:][pad] = 0
    return out


def mut_ball_scan_order(ref, centres):
    """rows written in the order the centres are scanned (sorted by y) instead of at their own index"""
    order = np.argsort(centres[..., 1], axis=1, kind="stable")
    return np.take_along_axis(ref, order[..., None].repeat(ref.shape[2], -1), 1)


def fps_lowest_index(xyz, m, skip=True):
    """furthest-point sampling of one frame [n,3] whose arg-max takes the LOWEST index among equal distances (the
    reference's tree prefers the smallest bit-reversed thread id instead).  skip=False also drops the rule that points
    with |p|^2 <= 1e-3 are never chosen."""
    mag = (xyz.astype(np.float64) ** 2).sum(1)                  # eligibility only: the clouds keep away from 1e-3
    temp = np.where((mag <= 1e-3) & skip, F32(-1), F32(1e10)).astype(np.float32)
    out = np.zeros(m, np.int32)
    old = 0
    for j in range(1, m):
        d = pn2.sqdist(xyz[old:old + 1], xyz)[0]
        temp = np.where(temp < 0, temp, np.minimum(d, temp))
        old = int(np.argmax(temp)) if temp.max() >= 0 else 0
        out[j] = old
    return out


def gather_rows(x, idx):
    """x [B,n,3], idx [B,m] -> [B,m,3]"""
    return np.take_along_axis(x, idx[..., None].astype(np.int64).repeat(x.shape[2], -1), 1)
