"""ICP refinement on the GPU (csrc/icp.cu): the my_icp drop-in against goldens recorded from the
reference, exact nearest neighbours, the batched refiner against the NumPy oracle, selection and
skipping, accuracy, stream plumbing and determinism."""
import os

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from oracle import icp_oracle
from pvn3d_b200 import fixtures, synth
from pvn3d_b200.eval_utils import FramePoseSolver, pose_add_adds
from pvn3d_b200.icp import IcpRefiner, my_icp

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "icp_cases.npz")
TOL_T = 1e-9
TOL_D = 1e-9


def golden_cases():
    z = np.load(GOLDEN)
    for k, name in enumerate(z["names"]):
        p = f"c{k}_"
        yield (str(name), z[p + "A"], z[p + "B"], z[p + "init"] if bool(z[p + "has_init"]) else None,
               int(z[p + "max_iter"]), float(z[p + "tol"]), z[p + "T"], z[p + "dist"], int(z[p + "i"]))


def kd_nearest(q, pts, k=4):
    """exact nearest neighbours for the oracle on large batches: k-d tree candidates, then the same
    float64 distance and lowest-index tie rule as the brute force"""
    k = min(k, len(pts))
    _, cand = cKDTree(pts).query(q, k=k)
    cand = cand.reshape(len(q), k)
    d2 = ((q[:, None, :] - pts[cand]) ** 2).sum(-1)
    best = d2.min(1, keepdims=True)
    idx = np.where(d2 == best, cand, np.iinfo(np.int64).max).min(1)
    return np.sqrt(best[:, 0]), idx


@pytest.mark.parametrize("case", list(golden_cases()), ids=lambda c: c[0])
def test_my_icp_matches_reference(cuda_dev, case):
    name, A, B, init, it, tol, T, dist, i = case
    Tg, dg, ig = my_icp(A, B, init, max_iterations=it, tolerance=tol, device=cuda_dev)
    assert ig == i
    assert Tg.shape == (4, 4) and Tg.dtype == np.float64 and np.array_equal(Tg[3], [0, 0, 0, 1])
    assert np.abs(Tg - T).max() <= TOL_T, np.abs(Tg - T).max()
    assert dg.shape == dist.shape and np.abs(dg - dist).max() <= TOL_D


def test_my_icp_takes_tensors(cuda_dev):
    name, A, B, init, it, tol, T, dist, i = next(golden_cases())
    Tg, dg, ig = my_icp(torch.from_numpy(A).to(cuda_dev), torch.from_numpy(B), torch.from_numpy(init), it, tol,
                        device=cuda_dev)
    assert ig == i and np.abs(Tg - T).max() <= TOL_T


def _check_nn(model, queries, dev):
    _, d, i = my_icp(model, queries, None, max_iterations=1, tolerance=0.0, device=dev)
    want, _ = icp_oracle.nearest(queries.astype(np.float64), model.astype(np.float64))
    assert i == 0
    assert np.abs(d - want).max() <= 1e-12


def test_exact_nearest_neighbour(cuda_dev):
    rng = np.random.default_rng(5)
    model = synth.box_surface((0.10, 0.06, 0.03), 3000, rng)
    model = np.concatenate([model, model[:200]])                     # duplicate points
    lo, hi = model.min(0), model.max(0)
    inside = rng.uniform(lo - 0.01, hi + 0.01, size=(1500, 3))
    far = rng.normal(size=(300, 3)) * 2.0 + np.array([3.0, -1.0, 0.5])   # far outside the model's box
    # queries on a regular lattice through the box, and exactly on model points
    lat = np.stack(np.meshgrid(*[np.linspace(lo[d], hi[d], 9) for d in range(3)], indexing="ij"), -1).reshape(-1, 3)
    on_pts = model[rng.choice(len(model), 200)]
    q = np.concatenate([inside, far, lat, on_pts]).astype(np.float32)
    _check_nn(model, q, cuda_dev)


def test_nearest_neighbour_on_cell_faces(cuda_dev):
    # The grid's cell edge is a power of two and its origin a multiple of it.  A box with dyadic extents
    # centred at the origin, its points and the queries on multiples of 2^-9 m: for any cell edge of
    # 2^-9 m or more (this model gets 2^-8 m) the queries lie on cell faces in every axis, and
    # the model points sit on faces too, with many exact distance ties.
    rng = np.random.default_rng(7)
    q9 = 2.0 ** -9
    model = np.round(synth.box_surface((0.125, 0.0625, 0.03125), 3000, rng) / q9) * q9
    lo, hi = model.min(0) - 4 * q9, model.max(0) + 4 * q9
    axes = [np.arange(np.floor(lo[d] / q9), np.ceil(hi[d] / q9) + 1) * q9 for d in range(3)]
    lat = np.stack(np.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3)
    q = lat[rng.choice(len(lat), 6000, replace=False)]
    assert np.all(np.round(q / q9) * q9 == q) and np.all(np.round(model / q9) * q9 == model)
    _check_nn(model.astype(np.float32), q.astype(np.float32), cuda_dev)


def test_nearest_neighbour_under_skewed_init(cuda_dev):
    # A float32 rotation promoted to float64 is not exactly orthogonal: the match must still be the
    # nearest point of src = init * A by the camera-frame distance, as a brute force over src finds it.
    rng = np.random.default_rng(8)
    model = synth.box_surface((0.10, 0.06, 0.03), 3000, rng)
    R = synth._haar_rotation(rng).astype(np.float32).astype(np.float64)
    R += rng.normal(0.0, 1e-6, (3, 3))                   # 1e-6 skew, well above float32's
    init = np.eye(4)
    init[:3, :3], init[:3, 3] = R, [0.02, -0.01, 0.7]
    src = model.astype(np.float64) @ R.T + init[:3, 3]
    q = (src[rng.choice(len(src), 1500)] + rng.normal(0, 0.002, (1500, 3))).astype(np.float32)
    _, d, i = my_icp(model, q, init, max_iterations=1, tolerance=0.0, device=cuda_dev)
    want, _ = icp_oracle.nearest(q.astype(np.float64), src)
    assert i == 0 and np.abs(d - want).max() <= 1e-12


def test_default_device_and_build_on_another_stream(cuda_dev):
    data = synth.make_icp_batch(2, 3, 600, seed=9, n_bg=200)
    t = {k: torch.from_numpy(np.ascontiguousarray(data[k])).to(cuda_dev) for k in ("pcld", "mask", "init", "present")}
    b, n, _ = data["pcld"].shape
    want = [o.clone() for o in _refiner(2, data, cuda_dev, max_pts=500, min_pts=100).refine(
        t["pcld"], t["mask"], t["init"], t["present"])]
    torch.cuda.synchronize()
    s_build, s_run = torch.cuda.Stream(cuda_dev), torch.cuda.Stream(cuda_dev)
    with torch.cuda.stream(s_build):                   # device="cuda" (no index), built on one stream ...
        ref = IcpRefiner(data["models"], len(data["models"]), b, n, max_pts=500, min_pts=100)
    assert ref.dev == t["pcld"].device
    s_run.wait_stream(torch.cuda.current_stream(cuda_dev))
    with torch.cuda.stream(s_run):                     # ... and used at once on another
        got = ref.refine(t["pcld"], t["mask"], t["init"], t["present"])
    torch.cuda.synchronize()
    for a, g in zip(want, got):
        assert torch.equal(a, g)


def test_nearest_neighbour_tiny_models(cuda_dev):
    rng = np.random.default_rng(6)
    q = rng.normal(size=(500, 3)).astype(np.float32)
    _check_nn(np.array([[0.1, -0.2, 0.3]], np.float32), q, cuda_dev)
    _check_nn(np.array([[0.1, -0.2, 0.3], [0.1, -0.2, 0.35]], np.float32), q, cuda_dev)
    _check_nn(np.array([[0.0, 0.0, 0.0], [0.0, 0.0, 0.0]], np.float32), q, cuda_dev)       # exact duplicates
    flat = np.column_stack([rng.uniform(0, 0.1, 400), rng.uniform(0, 0.05, 400), np.zeros(400)]).astype(np.float32)
    _check_nn(flat, q * 0.05, cuda_dev)


def _refiner(batch, data, dev, **kw):
    b, n, _ = data["pcld"].shape
    return IcpRefiner(data["models"], len(data["models"]), b, n, device=dev, **kw)


def _run(ref, data, dev, present=None):
    t = lambda k: torch.from_numpy(np.ascontiguousarray(data[k])).to(dev)
    pres = t("present") if present is None else torch.from_numpy(present).to(dev)
    out = ref.refine(t("pcld"), t("mask"), t("init"), pres)
    return [o.cpu().numpy() for o in out]


def _oracle_fit(data, b, c, max_pts, max_iter, tol):
    sel = icp_oracle.select(data["mask"][b], c, max_pts)
    init = np.eye(4)
    init[:3] = data["init"][b, c].astype(np.float64)
    return icp_oracle.my_icp(data["models"][c], data["pcld"][b][sel], init, max_iter, tol, nn=kd_nearest)


@pytest.fixture(scope="module")
def ycb_batch():
    return synth.make_icp_batch(16, 5, 2500, seed=11, outlier_frac=0.10)


def test_batched_matches_oracle(cuda_dev, ycb_batch):
    data = ycb_batch
    ref = _refiner(16, data, cuda_dev, max_pts=2000, min_pts=1500)
    poses, iters, err, refined = _run(ref, data, cuda_dev)
    assert poses.dtype == np.float64 and iters.dtype == np.int32 and refined.dtype == np.uint8
    n_fit = 0
    for b in range(16):
        for c in range(ref.n_cls):
            if not data["present"][b, c]:
                assert refined[b, c] == 0
                continue
            assert refined[b, c] == 1
            T, d, i = _oracle_fit(data, b, c, 2000, 500, 1e-9)
            assert iters[b, c] == i, (b, c, iters[b, c], i)
            assert np.abs(poses[b, c] - T[:3]).max() <= TOL_T
            assert abs(err[b, c] - d.mean()) <= TOL_D
            n_fit += 1
    assert n_fit == 80


def test_selection_and_skipping(cuda_dev):
    data = synth.make_icp_batch(3, 4, 300, seed=3, n_bg=300)
    mask = data["mask"]
    b0 = 0
    c_few = int(np.nonzero(data["present"][b0])[0][0])
    few = np.nonzero(mask[b0] == c_few)[0]
    mask[b0, few[100:]] = 0                                  # 100 points left: below min_pts
    present = data["present"].copy()
    present[:, 0] = 1                                        # class 0 is never refined, whatever the flag
    c_abs = int(np.nonzero(data["present"][1] == 0)[0][1])
    ref = _refiner(3, data, cuda_dev, max_pts=250, min_pts=150, max_iter=100, tol=1e-9)
    poses, iters, err, refined = _run(ref, data, cuda_dev, present=present)
    init64 = data["init"].astype(np.float64)
    for b in range(3):
        for c in range(ref.n_cls):
            skip = c == 0 or not data["present"][b, c] or (b == b0 and c == c_few)
            if skip:
                assert refined[b, c] == 0 and iters[b, c] == 0
                assert np.array_equal(poses[b, c], init64[b, c])  # passed through exactly
            else:
                assert refined[b, c] == 1
                assert (mask[b] == c).sum() == 300             # > max_pts: the strided subset is used
                T, d, i = _oracle_fit(data, b, c, 250, 100, 1e-9)
                assert iters[b, c] == i and np.abs(poses[b, c] - T[:3]).max() <= TOL_T
    assert refined[1, c_abs] == 0


def test_refinement_lowers_add(cuda_dev):
    data = synth.make_icp_batch(8, 5, 1500, seed=21, noise=0.001, angle_deg=5.0, offset=0.01)
    ref = _refiner(8, data, cuda_dev, max_pts=2000, min_pts=500)
    poses, iters, err, refined = _run(ref, data, cuda_dev)
    bound = 3e-3   # 3x the 1 mm point noise
    for b in range(8):
        for c in np.nonzero(data["present"][b])[0]:
            assert refined[b, c] == 1
            mdl = torch.from_numpy(data["models"][c]).to(cuda_dev)
            gt = torch.from_numpy(data["gt"][b, c]).to(cuda_dev)
            before = float(pose_add_adds(torch.from_numpy(data["init"][b, c]).to(cuda_dev), gt, mdl)[0][0])
            after = float(pose_add_adds(torch.from_numpy(poses[b, c]).to(cuda_dev), gt, mdl)[0][0])
            assert after < before and after < bound, (b, c, before, after)


def _placeholder_models(n_cls, rng):
    return {c: synth.box_surface(rng.uniform(0.04, 0.1, 3), 800, rng) for c in range(1, n_cls) if c % 4 != 3}


def test_chains_after_frame_pose_solver(cuda_dev):
    frames = synth.make_batch("ycb", 4)
    st = synth.stack(frames)
    b, n = st["pcld"].shape[:2]
    n_cls = fixtures.YCB_N_CLASSES
    solver = FramePoseSolver(b, n, fixtures.N_KEYPOINTS, n_cls, fixtures.mesh_kps_table_ycb(),
                             fixtures.radius_thresholds_ycb(), True, device=cuda_dev)
    ref = IcpRefiner(_placeholder_models(n_cls, np.random.default_rng(0)), n_cls, b, n, max_pts=400, min_pts=50,
                     max_iter=30, tol=1e-9, device=cuda_dev)
    d = {k: torch.from_numpy(v).to(cuda_dev) for k, v in st.items()}
    poses, present, _, new_mask = solver.solve(d["pcld"], d["labels"], d["ctr_of"], d["kp_of"])
    rp, it, err, refined = ref.refine(d["pcld"], new_mask, poses, present)
    assert rp.shape == (b, n_cls, 3, 4) and rp.dtype == torch.float64
    assert it.shape == (b, n_cls) and it.dtype == torch.int32
    assert err.dtype == torch.float64 and refined.dtype == torch.uint8
    torch.cuda.synchronize()
    pres = present.cpu().bool()
    assert pres.any()
    absent = ~pres
    assert torch.equal(rp.cpu()[absent], poses.cpu().double()[absent])
    assert not refined.cpu()[absent].any()
    has_model = torch.tensor([c % 4 != 3 and c > 0 for c in range(n_cls)])
    assert not refined.cpu()[:, ~has_model].any()
    assert refined.cpu()[pres & has_model[None]].any()


def test_refine_makes_no_host_sync(cuda_dev):
    data = synth.make_icp_batch(2, 3, 400, seed=4, n_bg=200)
    ref = _refiner(2, data, cuda_dev, max_pts=300, min_pts=100)
    t = {k: torch.from_numpy(np.ascontiguousarray(data[k])).to(cuda_dev) for k in ("pcld", "mask", "init", "present")}
    ref.refine(t["pcld"], t["mask"], t["init"], t["present"])          # warm
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        ref.refine(t["pcld"], t["mask"], t["init"], t["present"])
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    torch.cuda.synchronize()


def test_refine_on_side_stream_and_determinism(cuda_dev):
    data = synth.make_icp_batch(4, 5, 1200, seed=8, outlier_frac=0.1)
    ref = _refiner(4, data, cuda_dev, max_pts=1000, min_pts=500)
    first = _run(ref, data, cuda_dev)
    again = _run(ref, data, cuda_dev)
    for a, b in zip(first, again):
        assert np.array_equal(a, b)                                   # bit-identical run to run
    t = {k: torch.from_numpy(np.ascontiguousarray(data[k])).to(cuda_dev) for k in ("pcld", "mask", "init", "present")}
    torch.cuda.synchronize()
    s = torch.cuda.Stream(cuda_dev)
    with torch.cuda.stream(s):
        ref.poses.fill_(float("nan"))
        out = ref.refine(t["pcld"], t["mask"], t["init"], t["present"])
        done = torch.cuda.Event()
        done.record(s)
    done.synchronize()
    for a, b in zip(first, out):
        assert np.array_equal(a, b.cpu().numpy())
