"""Edge cases of csrc/icp.cu's model grid, nearest-neighbour search and fit, checked in float64.

- `grid(A)` restates icp_build_kernel's grid choice in numpy with the kernel's operations: the bounding box, the
  1e-3 * emax floor, target = min(16384, 4 * np), the power-of-two edge exp2(rint(log2(cbrt(...)))), the doubling
  loop, the per-cell counts, the Chebyshev distance transform (true and capped at 255) and the bound margin.  The
  host tests use it to show that each named case reaches the branch it is named for.
- `model(name)` / `queries(name, ...)` build the models and the queries the GPU tests search.
- `Reference` is icp_oracle's my_icp with its parts exposed: the nearest-neighbour rule, the per-step Kabsch, the
  stop rule, the final fit and the batched selection.  `ORACLE` is the plain one; `MUTANTS` are wrong references,
  each differing from it in one part, with the case the GPU tests catch it on.
"""
from __future__ import annotations

import numpy as np
import torch
from scipy import ndimage

from oracle import icp_oracle
from pvn3d_b200 import synth

MAX_CELLS = 16384   # kMaxCells
DT_CAP = 255        # the capped Chebyshev transform's uint8 ceiling


# ------------------------------------------------------------------------------------------------------------
# icp_build_kernel's grid, restated
# ------------------------------------------------------------------------------------------------------------
def grid(A) -> dict:
    a = np.asarray(A, np.float32).astype(np.float64)
    n = len(a)
    lo, hi = a.min(0), a.max(0)
    ext = hi - lo
    emax = max(0.0, float(ext.max()))
    floor_e = 1e-3 * emax + 1e-9
    e = np.maximum(ext, floor_e)
    target = min(float(MAX_CELLS), 4.0 * n)
    cell0 = float(np.exp2(np.rint(np.log2(np.cbrt(e[0] * e[1] * e[2] / target)))))
    cell, doublings = cell0, 0
    while True:
        glo = np.floor(lo / cell) * cell
        gdim = np.floor((hi - glo) / cell) + 1.0
        if gdim[0] * gdim[1] * gdim[2] <= MAX_CELLS:
            break
        cell *= 2.0
        doublings += 1
    dims = gdim.astype(np.int64)
    cmax = float(np.max(np.maximum(np.abs(glo), np.abs(glo + dims * cell))))
    cells = cell_index(a, glo, cell, dims)
    counts = np.bincount(cells, minlength=int(dims.prod()))
    occupied = counts.reshape(dims[::-1]) > 0                    # [z, y, x], the kernel's cell order
    dt_true = ndimage.distance_transform_cdt(~occupied, metric="chessboard").reshape(-1)
    return dict(lo=glo, h=cell, dims=dims, margin=1e-6 * cell + 1e-13 * cmax, target=target, cell0=cell0,
                doublings=doublings, floor_e=floor_e, emax=emax, counts=counts, dt_true=dt_true,
                dt=np.minimum(dt_true, DT_CAP))


def cell_index(q, lo, h, dims) -> np.ndarray:
    """the (clamped) cell of each point or query, as floor((x - lo) / h) clamped to [0, dims - 1]"""
    f = np.floor((np.asarray(q, np.float64) - lo) / h)
    c = np.clip(f, 0, dims - 1).astype(np.int64)
    return (c[:, 2] * dims[1] + c[:, 1]) * dims[0] + c[:, 0]


# ------------------------------------------------------------------------------------------------------------
# models
# ------------------------------------------------------------------------------------------------------------
OFFSET = np.array([50.0, -30.0, 80.0])
BOX = (0.10, 0.06, 0.03)
SIZES = {"pts_1": 1, "pts_3": 3, "pts_4095": 4095, "pts_4096": 4096, "cap_4097": 4097, "pts_16384": 16384,
         "pts_65536": 65536}
SHAPES = ("rod", "gap_600", "plane", "line", "outlier_10m", "offset_50m", "dups_40")
NAMES = tuple(SIZES) + SHAPES
# the rank of the model's spread: the final fit best_fit_transform(A, src) has a unique rotation only at rank >= 2
RANK_DEFICIENT = ("pts_1", "line")


def model(name: str) -> np.ndarray:
    """[P,3] float32 object-frame points of the named case"""
    rng = np.random.default_rng(NAMES.index(name) + 101)
    if name in SIZES:
        n = SIZES[name]
        if n < 4:
            return (np.array([[0.01, -0.02, 0.03], [0.05, 0.01, -0.02], [-0.03, 0.04, 0.01]])[:n]).astype(np.float32)
        return synth.box_surface(BOX, n, rng)
    if name == "rod":        # 1 m x 1 mm x 1 mm: the 1e-3 floor's first grid is over 16384 cells and doubles
        return (rng.uniform(0, 1, (4000, 3)) * [1.0, 1e-3, 1e-3]).astype(np.float32)
    if name == "gap_600":    # two 2 cm pieces of such a rod, 1 m apart: ~1000 empty cells between them
        p = rng.uniform(0, 1, (4000, 3)) * [0.02, 1e-3, 1e-3]
        p[2000:, 0] += 1.0
        return p.astype(np.float32)
    if name == "plane":      # zero width along z
        return np.column_stack([rng.uniform(0, 0.1, 4096), rng.uniform(0, 0.1, 4096),
                                np.full(4096, 0.05)]).astype(np.float32)
    if name == "line":       # a diagonal of the xy-plane: zero width along z, most cells of the grid empty
        t = rng.uniform(0, 0.1, 2000)
        return np.column_stack([t, t, np.full(2000, 0.02)]).astype(np.float32)
    if name == "outlier_10m":   # a 10 cm box inside one 0.25 m cell, and one point 10 m away
        box = synth.box_surface((0.1, 0.1, 0.1), 3000, rng).astype(np.float64) + 0.125
        far = 0.125 + 10.0 * np.ones(3) / np.sqrt(3.0)
        return np.concatenate([box, far[None]]).astype(np.float32)
    if name == "offset_50m":
        return (synth.box_surface(BOX, 3000, rng).astype(np.float64) + OFFSET).astype(np.float32)
    if name == "dups_40":    # 40 % of the points are exact copies of others, spread over the whole box
        p = synth.box_surface(BOX, 3000, rng)
        dst = rng.choice(3000, 1200, replace=False)
        src = rng.choice(np.setdiff1d(np.arange(3000), dst), 1200)
        p[dst] = p[src]
        return p
    raise KeyError(name)


def centre(A) -> np.ndarray:
    a = np.asarray(A, np.float64)
    return 0.5 * (a.min(0) + a.max(0))


def queries(name: str, A, faces: bool) -> dict:
    """named query sets (float32, object frame) around the model: inside its box, on dyadic cell faces (only when
    `faces`), outside each face and corner, in the middle of the rod's gap, and 100 m away"""
    rng = np.random.default_rng(NAMES.index(name) + 501)
    g = grid(A)
    a = np.asarray(A, np.float64)
    lo, hi = a.min(0), a.max(0)
    c, half = centre(a), 0.5 * (hi - lo)
    span = max(float((hi - lo).max()), 0.01)
    out = {"inside": rng.uniform(lo - 0.02 * span, hi + 0.02 * span, (1500, 3))}
    if faces:   # every coordinate on a cell face lo + k h (exact in float32 for these grids)
        k = rng.integers(-2, g["dims"] + 3, (800, 3))
        out["faces"] = g["lo"] + k * g["h"]
    dirs = np.array([(x, y, z) for x in (-1, 0, 1) for y in (-1, 0, 1) for z in (-1, 0, 1) if (x, y, z) != (0, 0, 0)])
    d = np.repeat(dirs, 12, 0)
    out["outside"] = c + d * (half + rng.uniform(0.05, 0.5, (len(d), 1)) * span) + \
        (d == 0) * rng.uniform(-1, 1, d.shape) * half
    if name == "gap_600":
        out["gap"] = np.column_stack([rng.uniform(0.45, 0.6, 300), rng.uniform(0, 1e-3, 300), rng.uniform(0, 1e-3, 300)])
    u = rng.normal(size=(100, 3))
    out["far_100m"] = c + 100.0 * u / np.linalg.norm(u, axis=1, keepdims=True)
    return {k: v.astype(np.float32) for k, v in out.items()}


def all_queries(name, A, faces) -> np.ndarray:
    return np.concatenate(list(queries(name, A, faces).values()))


# ------------------------------------------------------------------------------------------------------------
# poses
# ------------------------------------------------------------------------------------------------------------
def rot(axis, deg) -> np.ndarray:
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    a = np.deg2rad(deg)
    return np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K


def scene_pose(name: str) -> np.ndarray:
    """the pose G the scene is seen under: B = G q.  The offset box keeps its place (rotation about its centre)."""
    G = np.eye(4)
    G[:3, :3] = rot([0.3, -0.5, 0.8], 35.0)
    if name == "offset_50m":
        G[:3, 3] = OFFSET - G[:3, :3] @ OFFSET
    else:
        G[:3, 3] = [0.02, -0.01, 0.7]
    return G


INITS = ("rigid", "skew_1e-6", "scale_1.01", "shear_1e-3")


def init_pose(name: str, kind: str) -> np.ndarray:
    """4x4 float64 init near the scene pose: a rigid 2 degree / 1 mm error, a float32 rotation with 1e-6 skew,
    a 1.01 scale or a 1e-3 shear (the last three are not rigid: metric_shrink ~ 1 - 1e-6, 0.965, 0.9986)"""
    G = scene_pose(name)
    P = np.eye(4)
    P[:3, :3] = rot([1.0, 0.2, -0.4], 2.0) @ G[:3, :3]
    P[:3, 3] = G[:3, 3] + [0.001, -0.0005, 0.0007]
    if name == "offset_50m":     # keep the error a rotation about the model's centre
        P[:3, 3] = G[:3, :3] @ OFFSET + G[:3, 3] - P[:3, :3] @ OFFSET + [0.001, -0.0005, 0.0007]
    if kind == "skew_1e-6":
        P[:3, :3] = P[:3, :3].astype(np.float32).astype(np.float64) + \
            np.random.default_rng(3).normal(0.0, 1e-6, (3, 3))
    elif kind == "scale_1.01":
        P[:3, :3] = 1.01 * P[:3, :3]
    elif kind == "shear_1e-3":
        S = np.eye(3)
        S[0, 1] = 1e-3
        P[:3, :3] = P[:3, :3] @ S
    return P


def metric_shrink(P) -> float:
    """csrc/icp.cu's metric_shrink: 1 - ||M^T M - I||_F - 1e-12"""
    M = np.asarray(P, np.float64)[:3, :3]
    return max(0.0, 1.0 - float(np.linalg.norm(M.T @ M - np.eye(3))) - 1e-12)


def apply(P, X) -> np.ndarray:
    X = np.asarray(X, np.float64)
    return X @ np.asarray(P)[:3, :3].T + np.asarray(P)[:3, 3]


# ------------------------------------------------------------------------------------------------------------
# the float64 brute force, on whatever device the points are on
# ------------------------------------------------------------------------------------------------------------
def brute_nearest(q, pts, highest=False, f32=False, device="cpu", chunk=None):
    """exact nearest point of pts for every query: (distances, indices) as numpy.  One float64 op per step in
    numpy's order (dx*dx + dy*dy) + dz*dz, lowest index on ties (highest / float32 for the mutants)"""
    dt = torch.float32 if f32 else torch.float64
    qt = torch.as_tensor(np.asarray(q, np.float64), device=device).to(dt)
    pt = torch.as_tensor(np.asarray(pts, np.float64), device=device).to(dt)
    if highest:
        pt = pt.flip(0)
    n = len(pt)
    chunk = chunk or max(1, min(4096, (1 << 24) // max(n, 1)))
    d_out, i_out = [], []
    for s in range(0, len(qt), chunk):
        x = qt[s:s + chunk]
        dx = torch.sub(x[:, None, 0], pt[None, :, 0])
        dy = torch.sub(x[:, None, 1], pt[None, :, 1])
        dz = torch.sub(x[:, None, 2], pt[None, :, 2])
        d2 = torch.add(torch.add(torch.mul(dx, dx), torch.mul(dy, dy)), torch.mul(dz, dz))
        i = torch.argmin(d2, 1)
        d_out.append(torch.gather(d2, 1, i[:, None])[:, 0].double())
        i_out.append(i)
    d = np.sqrt(torch.cat(d_out).cpu().numpy())         # numpy's sqrt: torch's CPU one is not always rounded
    i = torch.cat(i_out).cpu().numpy().astype(np.int64)
    return d, (n - 1 - i if highest else i)


# ------------------------------------------------------------------------------------------------------------
# the reference and its mutants
# ------------------------------------------------------------------------------------------------------------
def fit_no_reflection_fix(A, B):
    ca, cb = A.mean(axis=0), B.mean(axis=0)
    U, _, Vt = np.linalg.svd((A - ca).T @ (B - cb))
    T = np.identity(4)
    T[:3, :3] = Vt.T @ U.T
    T[:3, 3] = cb - T[:3, :3] @ ca
    return T


def reflection_det(A, B) -> float:
    """det(V U^T) of best_fit_transform(A, B) before its reflection fix"""
    ca, cb = A.mean(axis=0), B.mean(axis=0)
    U, _, Vt = np.linalg.svd((A - ca).T @ (B - cb))
    return float(np.linalg.det(Vt.T @ U.T))


def select_round(mask_row, cls, max_pts):
    idx = np.nonzero(np.asarray(mask_row) == cls)[0]
    if len(idx) > max_pts:
        idx = idx[np.minimum(np.rint(np.arange(max_pts) * len(idx) / max_pts).astype(np.int64), len(idx) - 1)]
    return idx


class Reference:
    """icp_oracle.my_icp with its parts as attributes; `Reference()` computes exactly what icp_oracle.my_icp does"""

    def __init__(self, name="oracle", *, nn=None, step_fit=None, final_fit=None, stop=None, select=None,
                 model_frame=False, catches=None):
        self.name, self.catches = name, catches
        self.nn = nn or (lambda q, p, device: brute_nearest(q, p, device=device))
        self.step_fit = step_fit or icp_oracle.best_fit_transform
        self.final_fit = final_fit or (lambda A, B: icp_oracle.best_fit_transform(A, B))
        self.stop = stop or (lambda prev, mean, tol: np.abs(prev - mean) < tol)
        self.select = select or icp_oracle.select
        self.model_frame = model_frame

    def my_icp(self, A, B, init=None, max_iterations=20, tolerance=1e-3, device="cpu", trace=None):
        """icp_oracle.my_icp's loop; `trace`, a list, receives each step's mean distance"""
        A = np.asarray(A)
        B = np.asarray(B, np.float64)
        src = np.ones((4, len(A)))
        src[:3] = A.T
        P = np.identity(4) if init is None else np.asarray(init, np.float64)
        if init is not None:
            src = P @ src
        prev = 0.0
        for i in range(max_iterations):
            if self.model_frame:     # |P^-1 b - a| instead of |b - P a|
                q = apply(np.linalg.inv(P), B)
                distances, idx = self.nn(q, np.asarray(A, np.float64), device)
            else:
                distances, idx = self.nn(B, src[:3].T, device)
            T = self.step_fit(src[:3, idx].T, B)
            src = T @ src
            P = T @ P
            mean = np.mean(distances)
            if trace is not None:
                trace.append(mean)
            if self.stop(prev, mean, tolerance):
                break
            prev = mean
        return self.final_fit(A, src[:3].T), distances, i


ORACLE = Reference()
MUTANTS = {
    "tie_highest": Reference("tie_highest", nn=lambda q, p, device: brute_nearest(q, p, highest=True, device=device),
                             catches="dups_40 indices"),
    "dist_f32": Reference("dist_f32", nn=lambda q, p, device: brute_nearest(q, p, f32=True, device=device),
                          catches="pose-channel distances"),
    "model_frame": Reference("model_frame", model_frame=True, catches="scale_1.01 distances"),
    "select_round": Reference("select_round", select=select_round, catches="selection batch"),
    "stop_le": Reference("stop_le", stop=lambda prev, mean, tol: np.abs(prev - mean) <= tol,
                         catches="exact convergence, tol = 0"),
    "final_f64": Reference("final_f64", final_fit=lambda A, B: icp_oracle.best_fit_transform(
        np.asarray(A, np.float64), B), catches="offset_50m pose"),
    "no_reflection_fix": Reference("no_reflection_fix", step_fit=fit_no_reflection_fix,
                                   final_fit=fit_no_reflection_fix, catches="reflection plane pose"),
}


# ------------------------------------------------------------------------------------------------------------
# fit cases
# ------------------------------------------------------------------------------------------------------------
def box_model(seed=0, n=3000, extents=BOX) -> np.ndarray:
    return synth.box_surface(extents, n, np.random.default_rng(seed))


def fit_scene(A, seed, n=1500, noise=0.001, angle=5.0, offset=0.01):
    """(B [n,3] f32, init 4x4 f64): A's camera-facing points under a pose, and that pose perturbed"""
    rng = np.random.default_rng(seed)
    R = synth._haar_rotation(rng)
    t = np.array([0.02, -0.03, 0.8])
    ext = np.asarray(A, np.float64).max(0) - np.asarray(A, np.float64).min(0)
    B = synth.visible_box_points(ext, R, t, n, noise, rng)
    Ri, ti = synth.perturb_pose(R, t, angle, offset, rng)
    init = np.eye(4)
    init[:3, :3], init[:3, 3] = Ri, ti
    return B.astype(np.float32), init


def exact_scene():
    """a dyadic model, a dyadic signed-permutation pose and the scene init * A, exact in float32: every distance
    of step 0 is exactly 0, so mean = prev = 0 there"""
    rng = np.random.default_rng(41)
    pts = rng.permutation(np.unique(rng.integers(-64, 65, (3000, 3)), axis=0))[:2048] * 2.0 ** -10
    pts[:, 2] *= 0.5
    A = pts.astype(np.float32)
    init = np.eye(4)
    init[:3, :3] = [[0, -1, 0], [0, 0, 1], [-1, 0, 0]]
    init[:3, 3] = [0.25, -0.125, 0.75]
    B = apply(init, A)
    assert np.array_equal(B.astype(np.float32).astype(np.float64), B)
    return A, B.astype(np.float32), init


def rank_scenes():
    """max_iter = 1 fits of a full-rank box whose scene is degenerate: identical points (H = 0), collinear points
    (rank 1), and a plane (rank 2) whose SVD needs the reflection fix.  -> {name: (A, B, init)}"""
    A = box_model(seed=61)
    init = np.eye(4)
    init[:3, :3] = rot([0.2, 0.9, -0.3], 20.0)
    init[:3, 3] = [0.01, 0.02, 0.6]
    base = np.array([0.015625, -0.0078125, 0.609375])
    same = np.repeat(base[None], 256, 0)
    t = (np.arange(256) - 128) * 2.0 ** -11
    line = base + t[:, None] * np.array([1.0, 1.0, 1.0])
    out = {"identical": (A, same.astype(np.float32), init), "collinear": (A, line.astype(np.float32), init)}
    # a plane y = const in the camera frame, through the model; numpy's SVD of this H comes out with
    # det(V U^T) = -1, so the reflection fix decides R (asserted by the host tests)
    rng = np.random.default_rng(0)
    plane = rng.uniform(-0.05, 0.05, (512, 3)) + init[:3, 3]
    plane[:, 1] = np.float32(init[1, 3] + rng.uniform(-0.08, 0.08))
    out["plane_reflect"] = (A, plane.astype(np.float32), init)
    return out


def step_pieces(A, B, init, device="cpu"):
    """(src0 [P,3], idx) of step 0: init * A and the brute-force nearest of B in it"""
    src0 = (np.asarray(init) @ np.vstack([np.asarray(A, np.float64).T, np.ones(len(A))]))[:3].T
    _, idx = brute_nearest(np.asarray(B, np.float64), src0, device=device)
    return src0, idx


def undo_final_fit(A, P_out, rounds=4) -> np.ndarray:
    """P1 with best_fit_transform(A, P1 A) = P_out: the pose before my_icp's final fit.  That fit centres A in
    float32, which moves R and t by up to ~1e-10; the fixed point P <- P + (P_out - fit(P)) removes it."""
    P = np.array(P_out, np.float64)
    for _ in range(rounds):
        P = P + (P_out - icp_oracle.best_fit_transform(A, apply(P, A)))
    return P


def residual(T, X, B) -> float:
    return float((((apply(T, X) - np.asarray(B, np.float64)) ** 2).sum(-1)).sum())


# ------------------------------------------------------------------------------------------------------------
# batched selection and the mixed model buffer
# ------------------------------------------------------------------------------------------------------------
SEL_N, SEL_MAX, SEL_MIN = 12288, 1000, 200
SEL_COUNTS = {1: SEL_MIN - 1, 2: SEL_MIN, 3: SEL_MAX, 4: SEL_MAX + 1, 5: 2 * SEL_MAX + 1}   # frame 0
SEL_WHOLE = 6                                                                               # frame 1: every point
SEL_N_CLS = 8


def selection_batch() -> dict:
    rng = np.random.default_rng(71)
    extents, models = synth._box_models(SEL_N_CLS, 3000, rng)
    pcld = np.zeros((2, SEL_N, 3), np.float32)
    mask = np.zeros((2, SEL_N), np.int32)
    init = np.zeros((2, SEL_N_CLS, 3, 4), np.float32)
    init[:, :, :3, :3] = np.eye(3)
    present = np.zeros((2, SEL_N_CLS), np.uint8)
    rows = [dict(SEL_COUNTS), {SEL_WHOLE: SEL_N}]
    for b, counts in enumerate(rows):
        pts, lab = [], []
        for k, (c, cnt) in enumerate(counts.items()):
            R = synth._haar_rotation(rng)
            t = np.array([-0.3 + 0.15 * k, 0.05 * b, rng.uniform(0.6, 1.0)])
            pts.append(synth.visible_box_points(extents[c], R, t, cnt, 0.001, rng))
            lab.append(np.full(cnt, c, np.int32))
            Ri, ti = synth.perturb_pose(R, t, 5.0, 0.01, rng)
            init[b, c, :, :3], init[b, c, :, 3] = Ri, ti
            present[b, c] = 1
        n_bg = SEL_N - sum(counts.values())
        pts.append(np.column_stack([rng.uniform(-0.5, 0.5, (n_bg, 2)), np.full(n_bg, 1.2)]))
        lab.append(np.zeros(n_bg, np.int32))
        p, lb = np.concatenate(pts), np.concatenate(lab)
        order = rng.permutation(SEL_N)
        pcld[b], mask[b] = p[order], lb[order]
    present[0, 7] = 1          # present, but no point carries the class
    return dict(models=models, pcld=pcld, mask=mask, init=init, present=present)


MIX_N_CLS, MIX_B, MIX_N = 64, 36, 3000     # 36 * 64 = 2304 fits in one launch


def mixed_models() -> dict:
    """{class: points} for the 64-class refiner: None, one point, 4097 and 65536 points, the offset box, an empty
    array, and a box at the last class id; every other class has no entry"""
    return {1: None, 2: np.array([[0.01, 0.02, -0.01]], np.float32), 3: model("cap_4097"), 4: model("pts_65536"),
            5: model("offset_50m"), 6: np.zeros((0, 3), np.float32), 63: box_model(seed=63)}


def mixed_batch() -> dict:
    rng = np.random.default_rng(81)
    models = mixed_models()
    pcld = np.zeros((MIX_B, MIX_N, 3), np.float32)
    mask = np.zeros((MIX_B, MIX_N), np.int32)
    init = np.tile(np.eye(3, 4, dtype=np.float32), (MIX_B, MIX_N_CLS, 1, 1))
    init += rng.normal(0, 0.01, init.shape).astype(np.float32)          # passed through wherever skipped
    present = (rng.random((MIX_B, MIX_N_CLS)) < 0.5).astype(np.uint8)
    fit_cls = [2, 3, 4, 5, 63, 1, 6, 30]       # frames 0..7: one object each (the last three have no model)
    for b in range(MIX_B):
        p = np.column_stack([rng.uniform(-0.5, 0.5, (MIX_N, 2)), np.full(MIX_N, 1.2)])
        lab = np.zeros(MIX_N, np.int32)
        if b < len(fit_cls):
            c = fit_cls[b]
            A = np.asarray(models[c], np.float64) if models.get(c) is not None and len(models[c]) else box_model(b)
            ctr = centre(A)
            R = rot(rng.normal(size=3), 30.0)
            t = ctr + [0.0, 0.0, 0.3] if c == 5 else np.array([0.0, 0.0, 0.7])
            G = np.eye(4)
            G[:3, :3], G[:3, 3] = R, t - R @ ctr
            sel = rng.choice(len(A), 1500)
            p[:1500] = apply(G, A[sel]) + rng.normal(0, 0.001, (1500, 3))
            lab[:1500] = c
            Gi = np.eye(4)
            Gi[:3, :3] = rot(rng.normal(size=3), 3.0) @ R
            Gi[:3, 3] = t - Gi[:3, :3] @ ctr + rng.normal(0, 0.003, 3)
            init[b, c] = Gi[:3].astype(np.float32)
            present[b, c] = 1
        else:                                  # classes without a model, with points
            cs = rng.choice(np.arange(7, 63), 3, replace=False)
            lab[:900] = np.repeat(cs, 300)
        order = rng.permutation(MIX_N)
        pcld[b], mask[b] = p[order], lab[order]
    return dict(models=models, pcld=pcld, mask=mask, init=init, present=present, fit_cls=fit_cls)
