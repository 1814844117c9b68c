"""`pvn3d_best_fit_transform_batch` (float64 one-sided Jacobi SVD of kabsch.cuh, shared with ICP) against numpy's
float64 SVD of the same float32 inputs, and the pose solver's keypoint limit; plus `pose_add_adds` against a
float64 brute force at the edges of its 2048-point shared-memory tile.

Where the rotation is unique (the second singular value of H is well separated from the third, or all three are
positive and distinct) it must be within

    |R - R64|_F <= 1e-6 + 64 eps_32 * s_1 / gap

of numpy's, gap = the smallest difference between consecutive singular values (s_3 counts as such when it is
above zero), eps_32 = 2^-24: the float32 output rounds R to 2^-24, and a perturbation E of H moves the singular
vectors by |E| / gap.  Elsewhere (coplanar, collinear or coincident points; equal singular values) R must be a
rotation (orthonormal, det +1) whose residual equals numpy's optimum to 1e-6 relative.
"""
import numpy as np
import pytest
import torch

import ms_f64
from pvn3d_b200 import _lib, fixtures
from pvn3d_b200._lib import Pvn3dError, check, ptr
from pvn3d_b200.eval_utils import FramePoseSolver, pose_add_adds

pytestmark = pytest.mark.gpu
EPS32 = 2.0 ** -24


def _rot(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _shape(kind, p, rng):
    if kind == "random":
        return rng.normal(0, 0.1, (p, 3))
    if kind == "coplanar":
        return np.concatenate([rng.normal(0, 0.1, (p, 2)), np.zeros((p, 1))], 1)
    if kind == "collinear":
        return np.outer(rng.normal(0, 0.1, p), [0.3, -0.5, 0.8])
    if kind == "coincident":
        return np.zeros((p, 3))
    if kind == "cube":         # equal singular values
        c = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float64) * 0.05
        return c[np.arange(p) % 8]
    if kind == "tetra":
        c = np.array([[1, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1]], np.float64) * 0.05
        return c[np.arange(p) % 4]
    if kind == "near_equal":
        return rng.normal(0, 0.1, (p, 3)) * 1e-3 + _shape("cube", p, rng)
    raise ValueError(kind)


KINDS = ["random", "coplanar", "collinear", "coincident", "cube", "tetra", "near_equal"]
PS = [1, 2, 3, 4, 9, 32, 100]


def _cases(seed=0):
    """model points A, targets B = R A + t (+ noise, reflected, tiny or far), float32"""
    rng = np.random.default_rng(seed)
    A, B, tags = [], [], []
    for p in PS:
        for kind in KINDS:
            for variant in ("plain", "reflect", "tiny", "far"):
                a = _shape(kind, p, rng)
                if variant == "tiny":
                    a = a * 1e-3            # 1e-4 m scale
                R, t = _rot(rng), rng.normal(0, 0.3, 3)
                if variant == "far":
                    t = t + np.array([300.0, -120.0, 250.0])
                b = a @ R.T + t + rng.normal(0, 1e-3 * np.abs(a).max() if a.any() else 0.0, a.shape)
                if variant == "reflect":
                    b = b * np.array([1.0, 1.0, -1.0])
                A.append(a.astype(np.float32))
                B.append(b.astype(np.float32))
                tags.append((p, kind, variant))
    return A, B, tags


def _run_batch(A, B, valid, dev):
    p = A.shape[1]
    a, b = torch.from_numpy(A).to(dev), torch.from_numpy(B).to(dev)
    v = torch.from_numpy(valid.astype(np.uint8)).to(dev)
    rt = torch.full((len(A), 3, 4), float("nan"), dtype=torch.float32, device=dev)
    lib = _lib.load()
    rc = lib.pvn3d_best_fit_transform_batch(ptr(a), ptr(b), ptr(v), len(A), p, ptr(rt),
                                            torch.cuda.current_stream(dev).cuda_stream)
    check(rc, "pvn3d_best_fit_transform_batch")
    return rt.double().cpu().numpy()


def check_transform(a, b, rt, reflection_fix=True):
    """-> (ok, ratio, kind of check)"""
    R64, t64, s = ms_f64.kabsch_f64(a, b, reflection_fix)
    R, t = rt[:, :3], rt[:, 3]
    scale = max(float(s[0]), 1e-300)
    gaps = [s[0] - s[1], s[1] - s[2]] + ([s[2]] if s[2] > 1e-9 * scale else [])
    unique = s[1] > 1e-6 * scale and min(gaps) > 1e-6 * scale
    if unique:
        bound = 1e-6 + 64 * EPS32 * scale / min(gaps)
        ratio = float(np.linalg.norm(R - R64)) / bound
        return ratio <= 1.0, ratio, "unique"
    orth = float(np.abs(R @ R.T - np.eye(3)).max())
    det = float(np.linalg.det(R))
    if orth > 1e-6 or abs(det - 1.0) > 1e-6:
        return False, np.inf, "not a rotation"
    r_opt = ms_f64.kabsch_residual(a, b, R64, t64)
    a64, b64 = np.asarray(a, np.float64), np.asarray(b, np.float64)
    r_got = ms_f64.kabsch_residual(a, b, R, b64.mean(0) - R @ a64.mean(0))
    # 1e-6 of the optimum, plus what rounding R to float32 (|dR a| <= 4 eps_32 |a|) can add to it to first order
    ac = np.linalg.norm(a64 - a64.mean(0), axis=1)
    res = np.linalg.norm((a64 - a64.mean(0)) @ R64.T - (b64 - b64.mean(0)), axis=1)
    tol = 1e-6 * r_opt + float((8 * EPS32 * ac * (res + 4 * EPS32 * ac)).sum()) + 1e-30
    ratio = abs(r_got - r_opt) / tol
    return ratio <= 1.0, ratio, "residual"


def test_kabsch_against_numpy_float64(cuda_dev):
    A, B, tags = _cases()
    worst = {}
    for p in PS:
        sel = [i for i, tg in enumerate(tags) if tg[0] == p]
        # nfit across several 64-thread blocks, every other fit masked out
        reps = 3 if p <= 9 else 1
        idx = np.array(sel * reps)
        valid = np.arange(len(idx)) % 5 != 4
        rt = _run_batch(np.stack([A[i] for i in idx]), np.stack([B[i] for i in idx]), valid, cuda_dev)
        for j, i in enumerate(idx):
            if not valid[j]:
                assert np.array_equal(rt[j], np.eye(4)[:3]), "a masked fit is the identity"
                continue
            ok, ratio, kind = check_transform(A[i], B[i], rt[j])
            worst[kind] = max(worst.get(kind, 0.0), ratio)
            assert ok, (tags[i], kind, ratio)
            # the translation follows from R: t = mean(B) - R mean(A) (float32 output)
            a64, b64 = A[i].astype(np.float64), B[i].astype(np.float64)
            t_want = b64.mean(0) - rt[j, :, :3] @ a64.mean(0)
            assert np.linalg.norm(rt[j, :, 3] - t_want) <= 8 * EPS32 * (np.abs(b64).max() + np.abs(a64).max()) + 1e-9
    for k, v in sorted(worst.items()):
        print(f"F64RATIO kabsch/{k} {v:.4f}")
    assert set(worst) == {"unique", "residual"}


def test_kabsch_without_reflection_fix_is_caught(cuda_dev):
    A, B, tags = _cases(1)
    sel = [i for i, tg in enumerate(tags) if tg[1:] == ("random", "reflect") and tg[0] >= 4]
    rt = _run_batch(np.stack([A[i] for i in sel if len(A[i]) == 9]), np.stack([B[i] for i in sel if len(A[i]) == 9]),
                    np.ones(1, bool), cuda_dev)
    i = [k for k in sel if len(A[k]) == 9][0]
    assert check_transform(A[i], B[i], rt[0])[0]
    R_bad, _, _ = ms_f64.kabsch_f64(A[i], B[i], reflection_fix=False)
    assert np.linalg.det(R_bad) < 0
    assert np.linalg.norm(rt[0, :, :3] - R_bad) > 1e-3, "the reference without the fix must be rejected"


@pytest.mark.parametrize("k", [32, 33])
def test_solver_keypoint_limit(cuda_dev, k):
    """pose_kernel fits up to 32 keypoints + the centre; 33 is refused before anything is launched"""
    n, n_cls = 512, 3
    rng = np.random.default_rng(k)
    mesh = rng.normal(0, 0.05, (n_cls, k + 1, 3)).astype(np.float32)
    R, t = _rot(rng), np.array([0.05, -0.02, 0.8])
    s = FramePoseSolver(1, n, k, n_cls, mesh, None, False, device=cuda_dev)
    mask = np.zeros((1, n), np.int32)
    mask[0, :300] = 1
    pcld = rng.normal(0, 0.05, (1, n, 3)).astype(np.float32) + np.float32(0.8)
    targets = mesh[1] @ R.T + t
    ctr_of = (pcld[0] - targets[k]).astype(np.float32)[None]
    kp_of = (pcld[0][None] - targets[:k, None, :]).astype(np.float32)[None]
    args = [torch.from_numpy(np.ascontiguousarray(x)).to(cuda_dev) for x in (pcld, mask, ctr_of, kp_of)]
    if k == 33:
        with pytest.raises(Pvn3dError, match="unsupported"):
            s.solve(*args)
        return
    poses, present, cls_kps, _ = s.solve(*args)
    torch.cuda.synchronize()
    assert int(present[0, 1]) == 1
    got = poses[0, 1].double().cpu().numpy()
    R64, t64, _ = ms_f64.kabsch_f64(mesh[1], cls_kps[0, 1].cpu().numpy())
    assert np.linalg.norm(got[:, :3] - R64) <= 1e-5 and np.linalg.norm(got[:, 3] - t64) <= 1e-5
    assert np.linalg.norm(got[:, :3] - R) <= 1e-4


# ---- ADD / ADD-S -------------------------------------------------------------------------------
def _add_adds_f64(pr, gt, pts, dev):
    """float64 brute force on the device: (add [F], adds [F]) of float32 poses and points"""
    P = torch.from_numpy(pts.astype(np.float64)).to(dev)
    add, adds = [], []
    step = max(1, (1 << 24) // (2048 * len(pts)))      # one [step, 2048, P] float64 matrix stays <= 128 MiB
    for f0 in range(0, len(pr), step):
        r = torch.from_numpy(pr[f0:f0 + step].astype(np.float64)).to(dev)
        g = torch.from_numpy(gt[f0:f0 + step].astype(np.float64)).to(dev)
        pd = P @ r[:, :, :3].transpose(1, 2) + r[:, None, :, 3] - g[:, None, :, 3]     # centred on the gt translation
        gp = P @ g[:, :, :3].transpose(1, 2)
        add.append(torch.linalg.vector_norm(pd - gp, dim=-1).mean(1))
        nn = torch.cat([((g2 * g2).sum(-1)[:, :, None] + (pd * pd).sum(-1)[:, None, :]
                         - 2 * torch.bmm(g2, pd.transpose(1, 2))).amin(-1)
                        for g2 in gp.split(2048, dim=1)], 1)                 # rows of 2048 ground-truth points
        adds.append(nn.clamp(min=0).sqrt().mean(1))
    return torch.cat(add).cpu().numpy(), torch.cat(adds).cpu().numpy()


@pytest.mark.parametrize("p", [1, 255, 256, 2047, 2048, 2049, 4097, 7001])
def test_add_adds_against_float64(cuda_dev, p):
    """thread per ground-truth point, the predicted mesh streamed in 2048-point tiles; fixed-order sums"""
    rng = np.random.default_rng(p)
    pts = rng.uniform(-0.1, 0.1, (p, 3)).astype(np.float32)
    for f in (1, 63, 64, 65, 300):
        gt = np.zeros((f, 3, 4))
        pr = np.zeros((f, 3, 4))
        for i in range(f):
            gt[i, :, :3], gt[i, :, 3] = _rot(rng), rng.normal(0, 0.2, 3) + [0, 0, 0.8]
            v = rng.normal(0, 0.05, 3)
            th = np.linalg.norm(v)
            kx = np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]]) / th
            pr[i, :, :3] = (np.eye(3) + np.sin(th) * kx + (1 - np.cos(th)) * kx @ kx) @ gt[i, :, :3]
            pr[i, :, 3] = gt[i, :, 3] + rng.normal(0, 0.01, 3)
        pr32, gt32 = pr.astype(np.float32), gt.astype(np.float32)
        add, adds = pose_add_adds(torch.from_numpy(pr32).to(cuda_dev), torch.from_numpy(gt32).to(cuda_dev),
                                  torch.from_numpy(pts).to(cuda_dev))
        add, adds = add.double().cpu().numpy(), adds.double().cpu().numpy()
        add64, adds64 = _add_adds_f64(pr32, gt32, pts, cuda_dev)
        # float32 transforms of coordinates <= ~1.5 m: each distance is off by <= ~16 ulp(1.5) = 2e-6 m, the sums
        # and the mean add 1e-5 relative
        assert np.all(np.abs(add - add64) <= 2e-6 + 1e-5 * add64), (p, f, np.abs(add - add64).max())
        assert np.all(np.abs(adds - adds64) <= 2e-6 + 1e-5 * adds64), (p, f, np.abs(adds - adds64).max())
        # a tile dropped from the nearest-neighbour search would be caught: ADD-S over the first 2048 points only
        if p > 4096 and f == 1:
            P64 = pts.astype(np.float64)
            g = P64 @ gt32[0, :, :3].astype(np.float64).T
            d = P64[:2048] @ pr32[0, :, :3].astype(np.float64).T + (pr32[0, :, 3] - gt32[0, :, 3])
            wrong = np.sqrt(((g[:, None, :] - d[None]) ** 2).sum(-1).min(1)).mean()
            assert abs(adds[0] - wrong) > 2e-6 + 1e-5 * wrong
