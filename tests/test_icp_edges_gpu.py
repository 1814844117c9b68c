"""ICP refinement at its edges on the GPU (csrc/icp.cu) against the float64 oracle (tests/icp_edge_cases.py).

- Exact nearest neighbour on models that reach every branch of the grid build: 1 to 65536 points (the cell cap),
  a rod (the doubling loop), two clusters with a gap wider than the 255-cell transform, a plane and a line, a box
  with one point 10 m away, a box 100 m from the origin and 40 % duplicates.  Two channels reach nn_search: the
  label fill at the identity pose (indices bit-equal to a float64 brute force) and one my_icp step under a rigid,
  skewed, scaled or sheared init (distances within 1e-12, pose within 1e-9 of the oracle).
- The fit: class counts around min_pts / max_pts, a 64-class refiner with every kind of missing model, the C ABI's
  models buffer with fewer models than classes, the stop rule at i = 0, at the cap and at a tol equal to the
  oracle's own step, and rank-deficient Kabsch steps.
- The pruning budget of the search at the measured batch configuration.
- Each wrong reference of icp_edge_cases.MUTANTS fails the check the kernel passes, on the same data.

Runtime: 12-15 s for the module (four runs, H100 80GB HBM3 at 700 W).  Pair tests per query measured there: 7.07 at
the budgeted batch (DESIGN.md section 5c: 7.1), 1846 for outlier_10m and 88 for gap_600.
"""
import numpy as np
import pytest
import torch

import icp_edge_cases as E
from oracle import icp_oracle
from pvn3d_b200 import _lib, synth
from pvn3d_b200._lib import ptr
from pvn3d_b200.icp import IcpModels, IcpRefiner, _aligned, fill_label, my_icp

pytestmark = pytest.mark.gpu

TOL_D = 1e-12     # distances of one step
TOL_T = 1e-9      # poses
TOL_E = 1e-9      # mean distance of the batched fits


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


# ------------------------------------------------------------------------------------------------------------
# exact nearest neighbour: the identity channel (label fill, indices visible)
# ------------------------------------------------------------------------------------------------------------
def _fill(A, q, dev):
    lab = (np.arange(len(A), dtype=np.int64) * 7919 % 1000003).astype(np.int32)
    nn = torch.empty((1, len(q)), dtype=torch.int32, device=dev)
    got = fill_label(_t(q[None], dev), torch.ones((1, len(q)), dtype=torch.uint8, device=dev), _t(A[None], dev),
                     _t(lab[None], dev), nn_idx=nn)
    return nn[0].cpu().numpy(), got[0].cpu().numpy(), lab


def identity_failures(A, q, nn, labels, lab, ref, dev):
    _, want = ref.nn(q, A, dev)
    bad = []
    if not np.array_equal(nn, want):
        bad.append(f"{int((nn != want).sum())} indices differ")
    if not np.array_equal(labels, lab[want]):
        bad.append("labels differ")
    return bad


@pytest.mark.parametrize("name", E.NAMES)
def test_identity_channel_equals_brute_force(cuda_dev, name):
    A = E.model(name)
    q = E.all_queries(name, A, faces=True)
    nn, labels, lab = _fill(A, q, cuda_dev)
    assert not identity_failures(A, q, nn, labels, lab, E.ORACLE, cuda_dev)


def test_identity_channel_rejects_highest_index_on_ties(cuda_dev):
    A = E.model("dups_40")
    q = E.all_queries("dups_40", A, faces=True)
    nn, labels, lab = _fill(A, q, cuda_dev)
    assert not identity_failures(A, q, nn, labels, lab, E.ORACLE, cuda_dev)
    assert identity_failures(A, q, nn, labels, lab, E.MUTANTS["tie_highest"], cuda_dev)


# ------------------------------------------------------------------------------------------------------------
# exact nearest neighbour: the pose channel (one my_icp step under a non-identity init)
# ------------------------------------------------------------------------------------------------------------
def pose_case(name, kind):
    A = E.model(name)
    B = E.apply(E.scene_pose(name), E.all_queries(name, A, faces=False)).astype(np.float32)
    return A, B, E.init_pose(name, kind)


def step_failures(A, B, init, got, ref, dev, unique=True, max_iter=1, tol=0.0):
    T, d, i = got
    Tw, dw, iw = ref.my_icp(A, B, init, max_iter, tol, device=dev)
    bad = []
    if i != iw:
        bad.append(f"i {i} != {iw}")
    if not np.abs(d - dw).max() <= TOL_D:
        bad.append(f"distances off by {np.abs(d - dw).max():.3g}")
    if unique and not np.abs(T - Tw).max() <= TOL_T:
        bad.append(f"pose off by {np.abs(T - Tw).max():.3g}")
    return bad


def rotation_failures(R):
    bad = []
    if not (np.all(np.isfinite(R)) and np.abs(R.T @ R - np.eye(3)).max() <= 1e-12 and np.linalg.det(R) > 0):
        bad.append("not a rotation")
    return bad


@pytest.mark.parametrize("kind", E.INITS)
@pytest.mark.parametrize("name", E.NAMES)
def test_pose_channel_matches_oracle(cuda_dev, name, kind):
    A, B, init = pose_case(name, kind)
    got = my_icp(A, B, init, max_iterations=1, tolerance=0.0, device=cuda_dev)
    unique = name not in E.RANK_DEFICIENT
    assert not step_failures(A, B, init, got, E.ORACLE, cuda_dev, unique=unique)
    assert np.all(np.isfinite(got[0]))
    if not unique:          # a collinear or one-point model: the final fit's rotation is not unique
        assert not rotation_failures(got[0][:3, :3])


@pytest.mark.parametrize("mutant,name,kind", [("dist_f32", "pts_4096", "rigid"),
                                              ("model_frame", "pts_4096", "scale_1.01"),
                                              ("final_f64", "offset_50m", "rigid")])
def test_pose_channel_rejects_mutant(cuda_dev, mutant, name, kind):
    A, B, init = pose_case(name, kind)
    got = my_icp(A, B, init, max_iterations=1, tolerance=0.0, device=cuda_dev)
    assert not step_failures(A, B, init, got, E.ORACLE, cuda_dev)
    assert step_failures(A, B, init, got, E.MUTANTS[mutant], cuda_dev)


# ------------------------------------------------------------------------------------------------------------
# the batched fit: selection boundaries
# ------------------------------------------------------------------------------------------------------------
SEL_ITER = 100


def batch_failures(data, out, ref, dev, max_pts, min_pts, max_iter, tol=1e-9, models=None):
    """every fit of a batched refine() against ref, or its init passed through bit-exactly when skipped"""
    poses, iters, err, refined = out
    models = data["models"] if models is None else models
    b_n, n_cls = data["present"].shape
    bad, n_fit = [], 0
    for b in range(b_n):
        for c in range(n_cls):
            A = models[c] if isinstance(models, list) else models.get(c)
            has = A is not None and len(A) > 0
            cnt = int((data["mask"][b] == c).sum())
            init = np.eye(4)
            init[:3] = data["init"][b, c].astype(np.float64)
            if c == 0 or not data["present"][b, c] or not has or cnt < max(min_pts, 1):
                if refined[b, c] or iters[b, c] or not np.array_equal(poses[b, c], init[:3]):
                    bad.append(f"({b},{c}) not passed through")
                continue
            n_fit += 1
            sel = ref.select(data["mask"][b], c, max_pts)
            T, d, i = ref.my_icp(A, data["pcld"][b][sel], init, max_iter, tol, device=dev)
            if not refined[b, c] or iters[b, c] != i:
                bad.append(f"({b},{c}) iters {iters[b, c]} != {i}")
            elif not (np.abs(poses[b, c] - T[:3]).max() <= TOL_T and abs(err[b, c] - d.mean()) <= TOL_E):
                bad.append(f"({b},{c}) pose off by {np.abs(poses[b, c] - T[:3]).max():.3g}")
    return bad, n_fit


def _refine(ref, data, dev):
    out = ref.refine(_t(data["pcld"], dev), _t(data["mask"], dev), _t(data["init"], dev), _t(data["present"], dev))
    return [o.cpu().numpy() for o in out]


def test_selection_boundaries(cuda_dev):
    data = E.selection_batch()
    ref = IcpRefiner(data["models"], E.SEL_N_CLS, 2, E.SEL_N, max_pts=E.SEL_MAX, min_pts=E.SEL_MIN,
                     max_iter=SEL_ITER, tol=1e-9, device=cuda_dev)
    out = _refine(ref, data, cuda_dev)
    args = (cuda_dev, E.SEL_MAX, E.SEL_MIN, SEL_ITER)
    bad, n_fit = batch_failures(data, out, E.ORACLE, *args)
    assert not bad and n_fit == 5
    refined = out[3]
    assert refined[0].tolist() == [0, 0, 1, 1, 1, 1, 0, 0] and refined[1].tolist() == [0, 0, 0, 0, 0, 0, 1, 0]
    bad, _ = batch_failures(data, out, E.MUTANTS["select_round"], *args)
    assert len(bad) >= 3          # 1001, 2001 and 12288 points take the strided selection


# ------------------------------------------------------------------------------------------------------------
# the batched fit: a 64-class model buffer with every kind of missing model, and the C ABI's n_models < n_cls
# ------------------------------------------------------------------------------------------------------------
def test_mixed_model_buffer(cuda_dev):
    data = E.mixed_batch()
    assert E.MIX_B * E.MIX_N_CLS > 2048
    ref = IcpRefiner(data["models"], E.MIX_N_CLS, E.MIX_B, E.MIX_N, max_pts=1000, min_pts=100, max_iter=30,
                     tol=1e-9, device=cuda_dev)
    out = _refine(ref, data, cuda_dev)
    bad, n_fit = batch_failures(data, out, E.ORACLE, cuda_dev, 1000, 100, 30)
    assert not bad and n_fit == 5, bad
    refined = out[3]
    assert refined.sum() == 5 and all(refined[b, c] for b, c in enumerate(data["fit_cls"][:5]))


def test_cabi_skips_classes_beyond_the_models_buffer(cuda_dev):
    """pvn3d_icp_refine_batch on a models buffer built for 3 models while the mask has 8 classes: fits of
    classes 3..7 pass their init through (the kernel's c >= n_models rule, unreachable through model_table)"""
    rng = np.random.default_rng(91)
    n_cls, b_n, n = 8, 2, 4000
    A1, A2 = E.box_model(seed=1), E.box_model(seed=2, extents=(0.08, 0.05, 0.04))
    pts = np.concatenate([A1, A2])
    off = np.array([0, 0, len(A1), len(A1) + len(A2)], np.int32)
    models = IcpModels(pts, off, cuda_dev)
    pcld = np.zeros((b_n, n, 3), np.float32)
    mask = np.repeat(np.arange(n_cls, dtype=np.int32), n // n_cls)[None].repeat(b_n, 0)
    init = np.tile(np.eye(3, 4, dtype=np.float32), (b_n, n_cls, 1, 1))
    for b in range(b_n):
        for c in range(n_cls):
            B, ini = E.fit_scene(A1 if c != 2 else A2, seed=10 * b + c, n=n // n_cls)
            pcld[b, mask[b] == c] = B
            init[b, c] = ini[:3].astype(np.float32)
    present = np.ones((b_n, n_cls), np.uint8)
    lib = _lib.load()
    ws_bytes = int(lib.pvn3d_icp_workspace_bytes(b_n, n, n_cls, 400))
    ws, ws_ptr = _aligned(ws_bytes, cuda_dev)
    t = {k: _t(v, cuda_dev) for k, v in (("pcld", pcld), ("mask", mask), ("init", init), ("present", present))}
    poses = torch.empty((b_n, n_cls, 3, 4), dtype=torch.float64, device=cuda_dev)
    iters = torch.empty((b_n, n_cls), dtype=torch.int32, device=cuda_dev)
    err = torch.empty((b_n, n_cls), dtype=torch.float64, device=cuda_dev)
    refined = torch.empty((b_n, n_cls), dtype=torch.uint8, device=cuda_dev)
    with torch.cuda.device(cuda_dev):
        rc = lib.pvn3d_icp_refine_batch(models.ptr, ptr(t["pcld"]), ptr(t["mask"]), b_n, n, n_cls, ptr(t["init"]),
                                        ptr(t["present"]), 400, 100, 40, 1e-9, ptr(poses), ptr(iters), ptr(err),
                                        ptr(refined), ws_ptr, ws_bytes, torch.cuda.current_stream(cuda_dev).cuda_stream)
    _lib.check(rc, "pvn3d_icp_refine_batch")
    out = [x.cpu().numpy() for x in (poses, iters, err, refined)]
    data = dict(present=present, mask=mask, init=init, pcld=pcld)
    bad, n_fit = batch_failures(data, out, E.ORACLE, cuda_dev, 400, 100, 40, models={1: A1, 2: A2})
    assert not bad and n_fit == 4, bad
    assert out[3][:, 3:].sum() == 0 and out[3][:, 1:3].all()


# ------------------------------------------------------------------------------------------------------------
# the stop rule
# ------------------------------------------------------------------------------------------------------------
def test_stop_at_the_first_step_and_at_the_cap(cuda_dev):
    A = E.box_model(seed=5)
    B, init = E.fit_scene(A, seed=5)
    for it, tol, want_i in ((1, 1e-9, 0), (8, 0.0, 7)):
        got = my_icp(A, B, init, max_iterations=it, tolerance=tol, device=cuda_dev)
        assert got[2] == want_i
        assert not step_failures(A, B, init, got, E.ORACLE, cuda_dev, max_iter=it, tol=tol)


def test_exact_convergence_at_step_zero(cuda_dev):
    A, B, init = E.exact_scene()
    got = my_icp(A, B, init, max_iterations=5, tolerance=1e-9, device=cuda_dev)
    assert got[2] == 0 and np.all(got[1] == 0.0)
    assert not step_failures(A, B, init, got, E.ORACLE, cuda_dev, max_iter=5, tol=1e-9)
    got = my_icp(A, B, init, max_iterations=5, tolerance=0.0, device=cuda_dev)      # |0 - 0| < 0 is false
    assert got[2] == 4
    assert not step_failures(A, B, init, got, E.ORACLE, cuda_dev, max_iter=5, tol=0.0)
    assert step_failures(A, B, init, got, E.MUTANTS["stop_le"], cuda_dev, max_iter=5, tol=0.0)


@pytest.mark.parametrize("k", [2, 5])
def test_tol_equal_to_the_oracle_step(cuda_dev, k):
    A = E.box_model(seed=7)
    B, init = E.fit_scene(A, seed=7)
    means = []
    E.ORACLE.my_icp(A, B, init, 40, -1.0, device=cuda_dev, trace=means)
    steps = np.abs(np.diff(np.concatenate([[0.0], means])))
    tol = float(steps[k])
    assert np.all(steps[:k] > tol)            # the oracle does not stop before step k
    _, _, i_k = got = my_icp(A, B, init, max_iterations=40, tolerance=tol, device=cuda_dev)
    _, _, i_o = E.ORACLE.my_icp(A, B, init, 40, tol, device=cuda_dev)
    if i_k != i_o:                            # only a step whose difference equals tol to rounding may decide
        s = min(i_k, i_o)
        prev = means[s - 1] if s else 0.0
        assert abs(i_k - i_o) == 1 and abs(steps[s] - tol) <= 1e-12 * (prev + means[s]), (i_k, i_o)
    Tw, dw, iw = E.ORACLE.my_icp(A, B, init, i_k + 1, -1.0, device=cuda_dev)
    assert iw == i_k and np.abs(got[0] - Tw).max() <= TOL_T and np.abs(got[1] - dw).max() <= TOL_D


# ------------------------------------------------------------------------------------------------------------
# rank-deficient Kabsch steps
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scene", ["identical", "collinear", "plane_reflect"])
def test_rank_deficient_step(cuda_dev, scene):
    A, B, init = E.rank_scenes()[scene]
    got = my_icp(A, B, init, max_iterations=1, tolerance=0.0, device=cuda_dev)
    T, d, i = got
    assert np.all(np.isfinite(T)) and np.all(np.isfinite(d)) and i == 0
    if scene == "plane_reflect":              # rank 2: the reflection fix makes R unique
        assert not step_failures(A, B, init, got, E.ORACLE, cuda_dev)
        assert step_failures(A, B, init, got, E.MUTANTS["no_reflection_fix"], cuda_dev)
        return
    # rank 0 / 1: R is not unique; the step must be a rotation reaching numpy's optimal residual.  The returned
    # pose is the final fit of A to P1 A, whose float32 centring of A moves it by ~1e-10: undone first.
    assert not step_failures(A, B, init, got, E.ORACLE, cuda_dev, unique=False)
    step = E.undo_final_fit(A, T) @ np.linalg.inv(init)
    assert not rotation_failures(step[:3, :3])
    src0, idx = E.step_pieces(A, B, init, device=cuda_dev)
    best = E.residual(icp_oracle.best_fit_transform(src0[idx], B.astype(np.float64)), src0[idx], B)
    # 1e-12 relative, or an RMS residual within 1e-12 m where the optimum is 0 (identical points)
    assert abs(E.residual(step, src0[idx], B) - best) <= 1e-12 * best + len(B) * 1e-24


# ------------------------------------------------------------------------------------------------------------
# the search still prunes
# ------------------------------------------------------------------------------------------------------------
def test_pruning_budget(cuda_dev):
    """DESIGN.md section 5c's batch (tools/icp_bench.py at 5 deg / 1 cm): 7.1 pair tests per query measured; the
    count is deterministic for the seeded data, so 4x that bounds a search that has stopped pruning"""
    data = synth.make_icp_batch(16, 5, 2000, seed=105, model_pts=3000, angle_deg=5.0, offset=0.01)
    b, n, _ = data["pcld"].shape
    ref = IcpRefiner(data["models"], len(data["models"]), b, n, max_pts=2000, min_pts=1500, max_iter=500, tol=1e-9,
                     device=cuda_dev)
    _, iters, _, refined = _refine(ref, data, cuda_dev)
    queries = int(((iters[refined.astype(bool)] + 1) * 2000).sum())
    per_query = ref.pair_tests() / queries
    print(f"pair tests per query, 16 x 5 batch: {per_query:.2f}")
    assert int(refined.sum()) == 80 and per_query <= 28.0


@pytest.mark.parametrize("name", ["outlier_10m", "gap_600"])
def test_pair_tests_on_slow_cases(cuda_dev, name):
    """reported, not bounded: a box packed into one cell, and queries hundreds of empty cells from any point"""
    A = E.model(name)
    q = E.all_queries(name, A, faces=False)
    G = E.scene_pose(name)
    B = E.apply(G, q).astype(np.float32)
    ref = IcpRefiner({1: A}, 2, 1, len(B), max_pts=len(B), min_pts=1, max_iter=1, tol=0.0, device=cuda_dev)
    data = dict(pcld=B[None], mask=np.ones((1, len(B)), np.int32),
                init=np.stack([np.eye(3, 4), G[:3]]).astype(np.float32)[None], present=np.array([[0, 1]], np.uint8))
    _, iters, _, refined = _refine(ref, data, cuda_dev)
    assert refined[0, 1] == 1 and iters[0, 1] == 0
    print(f"pair tests per query, {name}: {ref.pair_tests() / len(B):.1f}")
