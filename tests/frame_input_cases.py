"""The inputs of tests/test_frame_input_edges_gpu.py: csrc/normals.cu at the edges of its sampler, its grid and its
exact 50-NN, with the mutants each case must tell from the reference (tests/normals_ref.py).

A mutant is a deliberately wrong restatement of an operation: something a kernel could compute instead.  A case is
a list of inputs plus the names of the mutants it must reject: the kernel has to equal the reference on every input
of the case, and every named mutant has to differ from the reference on at least one of them.  The second half needs
no GPU and is also run by tests/test_frame_input_cases_host.py.

Not a mutant: dividing the covariance by 49 instead of 50.  Eigenvectors and lambda0 / trace do not depend on the
scale of C, so no output of the kernel can tell the two apart.
"""
import functools

import numpy as np

import normals_ref as nr

F32 = np.float32
K = nr.K
SEEDS = (0, 1, 1 << 63, (1 << 64) - 1)


# ---- the sampler: sample_case(name) is dict(valid [B,hw] bool, n, seed, rgb_u8, labels, stride) -------------
SAMPLE_HW = (1000, 1024, 1025, 3 * 1024 + 7, 480 * 640)     # below, at and above one CTA's 1024-pixel stride
SAMPLE_N = (1, 50, 400, 12288)


def _nvs(hw, n):
    return sorted({v for v in (0, 1, 399, 400, 401, n - 1, n, n + 1, 2 * n, hw) if 0 <= v <= hw})


def _valid(hw, nvs, seed):
    rng = np.random.default_rng(seed)
    v = np.zeros((len(nvs), hw), bool)
    for f, nv in enumerate(nvs):
        if f % 3 == 2:
            v[f, hw - nv:] = True                   # packed at the end: the last, partial stride of the CTA
        else:
            v[f, rng.choice(hw, size=nv, replace=False)] = True
    return v


def _sample_cases():
    cases = {}
    i = 0
    for hw in SAMPLE_HW:
        for n in SAMPLE_N:
            # every combination of rgb dtype, labels and row stride appears among the 20 (hw, n) pairs
            cases[f"hw{hw}_n{n}"] = dict(valid=lambda hw=hw, n=n, i=i: _valid(hw, _nvs(hw, n), 10 + i), n=n,
                                         seed=SEEDS[i % 4], rgb_u8=i % 2, labels=(i // 2) % 2 == 0,
                                         stride=(9, 12)[(i // 4) % 2])
            i += 1
    # one launch of 72 frames: the frame index enters the key
    cases["b72"] = dict(valid=lambda: _valid(3079, [_nvs(3079, 400)[f % 7] for f in range(72)], 99), n=400,
                        seed=SEEDS[3], rgb_u8=1, labels=True, stride=12)
    return cases


SAMPLE_CASES = _sample_cases()


@functools.lru_cache(maxsize=None)
def sample_case(name):
    """SAMPLE_CASES[name] with its validity mask built"""
    case = dict(SAMPLE_CASES[name])
    case["valid"] = case["valid"]()
    return case


SAMPLE_MUTANTS = ("largest_keys", "key_b", "keep_n_minus_1", "keep_n_plus_1", "pad_edge", "pad_reflect", "ok_399",
                  "ok_401", "key_order")


def sample_data(case, seed=0):
    """(cloud [B,hw,3] f32, rgb [B,3,hw] u8 or f32, label_image [B,hw] i32 or None) for a sampler case.  Invalid
    pixels are NaN, so a wrongly chosen one cannot match; a few valid ones are -0.0 and subnormal (bit copies)."""
    valid = case["valid"]
    b, hw = valid.shape
    rng = np.random.default_rng(seed)
    cloud = rng.normal(size=(b, hw, 3)).astype(F32)
    cloud[:, ::97, 0] = F32(-0.0)
    cloud[:, 1::97, 1] = F32(1e-40)
    cloud[~valid] = np.nan
    if case["rgb_u8"]:
        rgb = rng.integers(0, 256, size=(b, 3, hw), dtype=np.uint8)
    else:
        rgb = rng.uniform(-300, 300, size=(b, 3, hw)).astype(F32)
    lab = rng.integers(-5, 1 << 20, size=(b, hw), dtype=np.int32) if case["labels"] else None
    return cloud, rgb, lab


def sample_rule(valid, n, seed, b, *, key_frame=None, largest=False, kept=None, pad="wrap",
                min_valid=nr.MIN_VALID, key_order=False):
    """(choose [n] i64, ok) of one frame under the sampling rule with its parts as parameters; the defaults are
    nr.sample_frame's.  key_frame: the frame index the key is seeded with; kept: how many of the smallest keys
    are taken (then wrapped or cut to n)."""
    valid = np.asarray(valid, bool).ravel()
    idx = np.nonzero(valid)[0]
    nv = len(idx)
    if nv < min_valid:
        return np.zeros(n, np.int64), 0
    if nv > n:
        keys = nr.sample_keys(seed, b if key_frame is None else key_frame, len(valid))[idx]
        order = np.argsort(keys, kind="stable")
        order = order[::-1] if largest else order
        take = order[: n if kept is None else kept]
        idx = idx[take] if key_order else np.sort(idx[take])
        if len(idx) >= n:
            return idx[:n].astype(np.int64), 1
        if len(idx) == 0:
            return np.zeros(n, np.int64), 1
    return np.pad(idx, (0, n - len(idx)), pad).astype(np.int64), 1


def sample_mutant(name, valid, n, seed, b):
    kw = {"largest_keys": dict(largest=True), "key_b": dict(key_frame=b - 1), "keep_n_minus_1": dict(kept=n - 1),
          "keep_n_plus_1": dict(kept=n + 1), "pad_edge": dict(pad="edge"), "pad_reflect": dict(pad="reflect"),
          "ok_399": dict(min_valid=399), "ok_401": dict(min_valid=401), "key_order": dict(key_order=True)}[name]
    return sample_rule(valid, n, seed, b, **kw)


def sample_ref(case, data):
    """what pvn3d_frame_sample must write: dict(choose [B,n] i64, ok [B] u8, cld6 [B,n,6] f32, labels [B,n] i32)"""
    cloud, rgb, lab = data
    valid, n = case["valid"], case["n"]
    b = len(valid)
    choose = np.zeros((b, n), np.int64)
    ok = np.zeros(b, np.uint8)
    cld6 = np.zeros((b, n, 6), F32)
    labels = np.zeros((b, n), np.int32)
    for f in range(b):
        choose[f], ok[f] = nr.sample_frame(valid[f], n, case["seed"], f)
        if ok[f]:
            cld6[f, :, :3] = cloud[f, choose[f]]
            cld6[f, :, 3:] = rgb[f][:, choose[f]].T.astype(F32)
            if lab is not None:
                labels[f] = lab[f, choose[f]]
    return dict(choose=choose, ok=ok, cld6=cld6, labels=labels)


def sample_mutant_differs(name, case, choose, ok):
    """does the mutant's (choose, ok) differ from the given one (the reference's, or the kernel's) on some frame"""
    valid, n, seed = case["valid"], case["n"], case["seed"]
    for f in range(len(valid)):
        c, o = sample_mutant(name, valid[f], n, seed, f)
        if o != ok[f] or not np.array_equal(c, choose[f]):
            return True
    return False


# ---- the neighbour sets: an input is (ref [B,R,3] f32, ref_valid [B,R] bool or None, query [B,Q,3] f32) ----------
def tie_cloud(seed, n=600):
    """dyadic lattice points (exact ties at equal distances), duplicates, and a few random points.  The lattice
    pitch is 1/8, so every power-of-two cell edge of at least 1/8 has its faces on lattice points."""
    rng = np.random.default_rng(seed)
    lat = rng.integers(-6, 7, size=(n // 2, 3)).astype(F32) / F32(8)
    dup = lat[rng.integers(0, len(lat), size=n // 4)]
    rnd = rng.normal(size=(n - len(lat) - len(dup), 3)).astype(F32)
    pts = np.concatenate([lat, dup, rnd])
    return pts[rng.permutation(len(pts))]


def _ties():
    ref = np.stack([tie_cloud(s) for s in (0, 1)])
    lat_q = np.random.default_rng(2).integers(-7, 8, size=(2, 200, 3)).astype(F32) / F32(8)
    return [(ref, None, np.concatenate([ref, lat_q], 1))]


def _coincident():
    rng = np.random.default_rng(3)
    pts = rng.normal(size=(300, 3)).astype(F32)
    pts[100:160] = pts[100]                                              # 60 copies: trace(C) = 0
    # "sampled" mode at n_v = 400: np.pad(..., 'wrap') of 400 samples to 12288, 30 or 31 copies of each
    wrap = np.resize(rng.normal(size=(400, 3)).astype(F32) * F32(0.05), (12288, 3))
    return [(pts[None], None, pts[None]), (wrap[None], None, np.ascontiguousarray(wrap[None, ::13]))]


def _counts():
    """frames with exactly 49, 50, 51 and 0 usable points beside a normal frame: the rest masked or non-finite"""
    rng = np.random.default_rng(4)
    r = 120
    ref = rng.normal(size=(5, r, 3)).astype(F32)
    valid = np.ones((5, r), bool)
    for f, k in ((0, 49), (1, 50), (2, 51), (3, 0)):
        cut = rng.permutation(r)[k:]
        valid[f, cut[: len(cut) // 2]] = False
        for j, i in enumerate(cut[len(cut) // 2:]):
            ref[f, i, j % 3] = (np.nan, np.inf, -np.inf)[j % 3]          # marked valid but not finite
    q = rng.normal(size=(5, 80, 3)).astype(F32)
    return [(ref, valid, q)]


def _nonfinite():
    rng = np.random.default_rng(5)
    ref = rng.uniform(-1, 1, size=(2, 400, 3)).astype(F32)
    ref[0, 5, 0], ref[0, 17, 1], ref[0, 33, 2], ref[1, 0] = np.nan, np.inf, -np.inf, np.nan
    ref[1, 399] = np.inf
    q = rng.uniform(-1, 1, size=(2, 100, 3)).astype(F32)
    q[:, :40] = ref[:, :40]                                              # on points, the non-finite ones included
    q[0, 50, 1], q[1, 60, 2], q[1, 61] = np.nan, -np.inf, np.inf
    return [(ref, None, q)]


def _outside():
    """queries just past each face of the reference box (one ulp, 1 mm) and 10^3 m away"""
    rng = np.random.default_rng(6)
    ref = rng.uniform(0, 1, size=(2, 1000, 3)).astype(F32)
    qs = []
    for f in range(2):
        lo, hi, mid = ref[f].min(0), ref[f].max(0), F32(0.5)
        q = []
        for d in range(3):
            for v in (np.nextafter(hi[d], F32(np.inf)), hi[d] + F32(1e-3), np.nextafter(lo[d], F32(-np.inf)),
                      lo[d] - F32(1e-3), F32(1e3), F32(-1e3)):
                p = np.full(3, mid, F32)
                p[d] = v
                q.append(p)
        q += [np.full(3, 1e3, F32), np.full(3, -1e3, F32), np.array([1e3, -1e3, 0.5], F32)]
        qs.append(np.concatenate([np.stack(q), ref[f, :20]]))
    return [(ref, None, np.stack(qs))]


def _extremes():
    """grids at their limits: a 300 m outlier (almost every point in one cell), a flat wall (a zero-width axis),
    a wall through the origin (n . p = 0), a line along x (lambda0 = lambda1 = 0), a 1e-4 m cloud, a cloud 300 m
    from the origin with mm spacing; and a frame of exactly R = 50 points"""
    rng = np.random.default_rng(7)
    r = 600
    out = rng.normal(scale=0.05, size=(r, 3))
    out[17] = (300.0, 0.0, 0.0)
    wall = np.c_[rng.uniform(-0.3, 0.3, size=(r, 2)), np.full(r, 0.7)]
    wall0 = np.c_[rng.uniform(-0.3, 0.3, size=(r, 2)), np.zeros(r)]
    line = np.c_[rng.uniform(-0.2, 0.2, r), np.full(r, 0.5), np.full(r, 0.25)]
    tiny = rng.uniform(0, 1e-4, size=(r, 3)) + 0.3
    far = rng.uniform(0, 0.05, size=(r, 3)) + (300.0, -2.0, 1.0)
    ref = np.stack([out, wall, wall0, line, tiny, far]).astype(F32)
    r50 = rng.normal(size=(1, 50, 3)).astype(F32)
    return [(ref, None, ref.copy()), (r50, None, np.concatenate([r50, rng.normal(size=(1, 30, 3)).astype(F32)], 1))]


def _scales():
    rng = np.random.default_rng(8)
    base = rng.uniform(-0.5, 0.5, size=(3, 800, 3))
    ref = (base * np.array([1e-3, 1.0, 1e2])[:, None, None] + (0.1, -0.2, 1.5)).astype(F32)
    return [(ref, None, ref[:, ::3].copy())]


def _d2_sum(d, assoc):
    d = d.astype(np.float64)
    s = d * d
    return s[..., 0] + (s[..., 1] + s[..., 2]) if assoc else (s[..., 0] + s[..., 1]) + s[..., 2]


def _twins():
    """query at the origin (each frame), and near it:
    * sub-ulp twins p1 = (s, 0, 0) and p2 = (s, s 2^-13, 0) at the lower index: their float64 d^2 differ, their
      float32 d^2 are equal;
    * order twins p and p' = p with its coordinates rotated, equidistant in exact arithmetic, chosen so that
      (dx^2 + dy^2) + dz^2 and dx^2 + (dy^2 + dz^2) order the pair strictly and oppositely (whatever their
      indices);
    then farther random points to fill the 50."""
    rng = np.random.default_rng(9)
    frames, queries = [], []
    for s in (1.0, 0.25, 3.0, 1.0):
        # coordinates of unlike magnitudes: their squares need more than 53 bits together
        p = (rng.normal(size=(20000, 3)) * 2.0 ** rng.uniform(-4, 0, size=(20000, 3))).astype(F32) * F32(s)
        pp = np.stack([p, np.roll(p, 1, axis=1)], 1)
        dc, dm = _d2_sum(pp, False), _d2_sum(pp, True)
        opp = (dc[:, 0] != dc[:, 1]) & (dm[:, 0] != dm[:, 1]) & ((dc[:, 0] < dc[:, 1]) != (dm[:, 0] < dm[:, 1]))
        opp &= dc[:, 0] < (2.5 * s) ** 2
        pairs = pp[np.nonzero(opp)[0][:10]]
        assert len(pairs) == 10
        sub = [np.array([s, s * 2.0 ** -13, 0.0], F32), np.array([s, 0.0, 0.0], F32)]   # lower index first
        fill = rng.normal(size=(200, 3)).astype(F32)
        fill = fill / np.linalg.norm(fill, axis=1, keepdims=True).astype(F32) * F32(6 * s)
        pts = np.concatenate([np.stack(sub), np.concatenate(pairs), fill]).astype(F32)
        perm = np.concatenate([[0, 1], 2 + rng.permutation(len(pts) - 2)])   # twins scattered, sub-ulp order kept
        frames.append(pts[perm])
        queries.append(np.concatenate([np.zeros((1, 3), F32), rng.normal(size=(15, 3)).astype(F32) * F32(s)]))
    return [(np.stack(frames), None, np.stack(queries))]


# name -> (inputs, kNN mutants, normal mutants) that the case must reject
KNN_CASES = {
    "ties": (_ties, ["highest_index", "no_self", "k49", "frame0", "cell27"],
             ["largest", "middle", "flip_reversed", "no_flip", "first32", "curv_lambda2"]),
    "coincident_wrap": (_coincident, ["highest_index", "no_self", "cell27"], ["trace0_nonzero", "first32"]),
    "usable_counts": (_counts, ["k49", "frame0", "admit_masked", "admit_nonfinite"], ["largest", "no_flip"]),
    "nonfinite": (_nonfinite, ["frame0", "no_self", "cell27"], ["middle", "flip_reversed"]),
    "outside": (_outside, ["frame0", "cell27"], ["largest", "flip_reversed"]),
    "extremes": (_extremes, ["no_self", "cell27"], ["one_pass", "largest", "flip_reversed"]),
    "scales": (_scales, ["frame0", "cell27"], ["largest", "middle", "first32", "curv_lambda2"]),
    "twins": (_twins, ["f32_distance", "assoc", "frame0"], ["largest", "first32"]),
}
KNN_MUTANTS = ("highest_index", "f32_distance", "assoc", "no_self", "k49", "frame0", "admit_masked",
               "admit_nonfinite", "cell27")
NORMAL_MUTANTS = ("one_pass", "largest", "middle", "flip_reversed", "no_flip", "trace0_nonzero", "first32",
                  "curv_lambda2")


def grid_rule(ref, valid, n_ref):
    """(lo [3], h, dims [3]) of one frame's search grid: a numpy restatement of grid_setup_kernel"""
    use = nr._usable(ref, valid)
    if len(use) == 0:
        return np.zeros(3), 1.0, np.ones(3, np.int64)
    p = np.asarray(ref, F32)[use].astype(np.float64)
    lo, hi = p.min(0), p.max(0)
    floor_e = 1e-3 * (hi - lo).max() + 1e-9
    e = np.maximum(hi - lo, floor_e)
    cap = 2 * n_ref + 64
    target = min(float(cap), 2.0 * len(use))
    cell = 2.0 ** np.rint(np.log2(np.cbrt(e[0] * e[1] * e[2] / target)))
    while True:
        glo = np.floor(lo / cell) * cell
        dims = np.floor((hi - glo) / cell) + 1.0
        if np.prod(dims) <= cap:
            return glo, cell, dims.astype(np.int64)
        cell *= 2.0


def _cell_of(p, lo, h, dims):
    with np.errstate(invalid="ignore"):
        f = np.floor((np.asarray(p, F32).astype(np.float64) - lo) / h)
    f = np.where(np.isfinite(f), f, 0)
    return np.clip(f, 0, dims - 1).astype(np.int64)


def knn_rule(ref, query, valid=None, *, dist="f64", tie="low", self_=True, k=K, admit_masked=False,
             admit_nonfinite=False, cell27=False):
    """[Q,50] int64 neighbour indices of one frame under the rule with its parts as parameters; the defaults are
    nr.knn_brute's.  Fewer than k admitted points, or a non-finite query, gives a -1 row; k < 50 leaves the
    last columns -1."""
    ref = np.asarray(ref, F32)
    ok = np.ones(len(ref), bool)
    if valid is not None and not admit_masked:
        ok &= np.asarray(valid, bool)
    if not admit_nonfinite:
        ok &= np.isfinite(ref).all(1)
    use = np.nonzero(ok)[0]
    out = np.full((len(query), K), -1, np.int64)
    if len(use) < k:
        return out
    if cell27:
        lo, h, dims = grid_rule(ref, valid, len(ref))
        cells = _cell_of(ref[use], lo, h, dims)
    for row, q in enumerate(np.asarray(query, F32)):
        if not np.isfinite(q).all():
            continue
        cand = use
        if cell27:
            near = (np.abs(cells - _cell_of(q[None], lo, h, dims)) <= 1).all(1)
            cand = use[near]
        d = q[None].astype(np.float64) - ref[cand].astype(np.float64)
        if dist == "f32":
            d = d.astype(F32)
            d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        else:
            with np.errstate(invalid="ignore"):
                d2 = _d2_sum(d, dist == "assoc")
        if not self_:
            keep = d2 != 0
            cand, d2 = cand[keep], d2[keep]
        sel = cand[np.lexsort((cand if tie == "low" else -cand, d2))][:k]
        out[row, : len(sel)] = sel
    return out


def knn_ref(inp):
    """[B,Q,50] int64: the reference (nr.knn) for every frame of an input"""
    ref, valid, q = inp
    return np.stack([nr.knn(ref[f], q[f], None if valid is None else valid[f]) for f in range(len(ref))])


def knn_mutant(name, inp):
    ref, valid, q = inp
    res = []
    for f in range(len(ref)):
        g = 0 if name == "frame0" else f
        v = None if valid is None else valid[g]
        kw = {"highest_index": dict(tie="high"), "f32_distance": dict(dist="f32"), "assoc": dict(dist="assoc"),
              "no_self": dict(self_=False), "k49": dict(k=K - 1), "frame0": {}, "admit_masked": dict(admit_masked=True),
              "admit_nonfinite": dict(admit_nonfinite=True), "cell27": dict(cell27=True)}[name]
        res.append(knn_rule(ref[g], q[f], v, **kw))
    return np.stack(res)


# ---- the normal of a neighbourhood ------------------------------------------------------------------------------
def normal_rule(ref, idx, query, *, cov="two_pass", which=0, flip="towards", trace0="zero", first=K,
                curv="trace"):
    """(n [Q,3] f64, curvature [Q]) of one frame's neighbour sets with the parts of the rule as parameters; the
    defaults are nr.normals'"""
    q = len(idx)
    n, cu = np.zeros((q, 3)), np.zeros(q)
    have = (idx >= 0).all(1)
    if not have.any():
        return n, cu
    p = np.asarray(ref, F32)[idx[have, :first]].astype(np.float64)
    m = p.mean(1, keepdims=True)
    if cov == "two_pass":
        C = np.einsum("qki,qkj->qij", p - m, p - m) / p.shape[1]
    else:                                                # E[p p^T] - mean mean^T
        C = np.einsum("qki,qkj->qij", p, p) / p.shape[1] - m[:, 0, :, None] * m[:, 0, None, :]
    w, v = np.linalg.eigh(C)
    nn = v[:, :, which].copy()
    tr = np.trace(C, axis1=1, axis2=2)
    qq = np.asarray(query, F32)[have].astype(np.float64)
    dot = (nn * qq).sum(1)
    if flip == "towards":
        nn[dot > 0] *= -1
    elif flip == "away":
        nn[dot < 0] *= -1
    zero = tr == 0
    if trace0 == "zero":
        nn[zero] = 0
    else:                                                # what Jacobi leaves for the zero matrix: column 0
        nn[zero] = np.where((qq[zero, :1] > 0), -1.0, 1.0) * np.array([1.0, 0.0, 0.0])
    n[have] = nn
    den = tr if curv == "trace" else w[:, 2]
    cu[have] = np.where(den > 0, np.maximum(w[:, 0], 0) / np.where(den > 0, den, 1), 0)
    return n, cu


def normal_mutant(name, ref, idx, query):
    kw = {"one_pass": dict(cov="one_pass"), "largest": dict(which=2), "middle": dict(which=1),
          "flip_reversed": dict(flip="away"), "no_flip": dict(flip="none"), "trace0_nonzero": dict(trace0="e_x"),
          "first32": dict(first=32), "curv_lambda2": dict(curv="lambda2")}[name]
    return normal_rule(ref, idx, query, **kw)


U64 = 2.0 ** -53     # unit roundoff of float64


def curvature_bound(want):
    """|got - want| allowed for the curvature lambda0 / trace of one neighbourhood.  The two sides compute C with
    different summation orders: each entry is a sum of 50 products of exactly centred coordinates (a common error
    in the mean enters only at second order, because the centred coordinates sum to zero), so each side's C is
    within gamma_50 * trace of the exact one entrywise, and its Frobenius norm within 3 gamma_50 * trace, gamma_50 ~
    50 u.  Both eigen-solvers are backward stable, within a few tens of u * ||C||.  By Weyl, each lambda0 / trace
    is then within ~200 u of the exact one: 512 u for the two sides with margin.  The float32 store adds half an
    ulp of the result, 2^-24 relative."""
    return 2.0 ** -24 * np.abs(want) + 512 * U64


def normal_faults(n, curv, C, lam, want, want_curv, q):
    """(names of the failed checks, worst values) of normals n [Q,3] f64 and curvature [Q] of one batch, flattened,
    against the reference's covariance C [Q,3,3], eigenvalues lam [Q,3], normal want [Q,3] and curvature, at the
    queries q [Q,3]:
      zero       trace(C) == 0 (no neighbourhood included) -> n and curvature exactly 0
      unit       | ||n|| - 1 | <= 1e-12
      residual   ||C n - lambda0 n|| <= 1e-9 trace(C)
      angle      <= 1e-6 rad to the reference where (lambda1 - lambda0) / trace >= 1e-3
      sign       n . q has the reference's sign where also |want . q| >= 1e-6 ||q||
      curvature  within curvature_bound"""
    n, curv, q = np.asarray(n, np.float64), np.asarray(curv, np.float64), np.asarray(q, F32).astype(np.float64)
    tr = np.trace(C, axis1=1, axis2=2)
    zero = tr == 0
    faults, worst = [], {}
    if n[zero].any() or curv[zero].any():
        faults.append("zero")
    g, Cz, l0, t, w, qq = n[~zero], C[~zero], lam[~zero, 0], tr[~zero], want[~zero], q[~zero]
    if g.size == 0:
        return faults, worst
    if not np.all(np.abs(np.linalg.norm(g, axis=1) - 1.0) <= 1e-12):
        faults.append("unit")
    res = np.linalg.norm(np.einsum("qij,qj->qi", Cz, g) - l0[:, None] * g, axis=1) / t
    worst["residual/trace"] = float(res.max())
    if not np.all(res <= 1e-9):
        faults.append("residual")
    sep = (lam[~zero, 1] - l0) / t >= 1e-3
    ang = np.arctan2(np.linalg.norm(np.cross(g[sep], w[sep]), axis=1), np.abs((g[sep] * w[sep]).sum(1)))
    worst["angle"] = float(ang.max()) if ang.size else 0.0
    if ang.size and ang.max() > 1e-6:
        faults.append("angle")
    clear = sep & (np.abs((w * qq).sum(1)) >= 1e-6 * np.linalg.norm(qq, axis=1))
    if not np.array_equal(np.sign((g[clear] * qq[clear]).sum(1)), np.sign((w[clear] * qq[clear]).sum(1))):
        faults.append("sign")
    err = np.abs(curv[~zero] - want_curv[~zero]) / curvature_bound(want_curv[~zero])
    worst["curvature/bound"] = float(err.max())
    if err.max() > 1.0:
        faults.append("curvature")
    return faults, worst


def normals_of(inp, idx):
    """the reference's (n, C, lam, curvature) of every frame of an input for neighbour sets idx [B,Q,50]"""
    ref, _, q = inp
    parts = [nr.normals(ref[f], idx[f], q[f]) for f in range(len(ref))]
    return tuple(np.concatenate([p[i] for p in parts]) for i in range(4))


def normal_mutant_faults(name, inp, idx):
    """the checks a normal mutant fails on an input, applied to the neighbour sets idx"""
    ref, _, q = inp
    n, C, lam, curv = normals_of(inp, idx)
    parts = [normal_mutant(name, ref[f], idx[f], q[f]) for f in range(len(ref))]
    mn, mc = np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
    return normal_faults(mn, mc, C, lam, n, curv, q.reshape(-1, 3))[0]
