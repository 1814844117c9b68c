"""The oracle against the reference's recorded outputs and against analytic known answers.

CPU only.  tests/golden/*.npz were produced by the reference itself (tests/golden/make_golden_cpu.py);
the KATs encode the semantics of SURVEY App. A that the reference's kernels implement.
"""
import os

import numpy as np
import pytest
import torch

from oracle import frame_poses_oracle, meanshift_oracle, pn2
from pvn3d_b200 import fixtures

MS_CASES = ["tight", "outl10", "outl30", "two", "wide", "bw002", "bw016", "single", "pair_far", "n1200"]


@pytest.mark.parametrize("name", MS_CASES)
def test_meanshift_oracle_matches_reference_bits(golden_dir, name):
    z = np.load(os.path.join(golden_dir, "ms_cases.npz"))
    if len(z[f"{name}_A"]) > 800:
        pytest.skip("large case covered on the GPU side (keeps the CPU suite fast)")
    orc = meanshift_oracle.MeanShiftOracle(bandwidth=float(z[f"{name}_bw"]))
    ctr, labels = orc.fit(torch.from_numpy(z[f"{name}_A"]))
    assert np.array_equal(ctr.numpy(), z[f"{name}_ctr"])
    assert np.array_equal(labels.numpy(), z[f"{name}_labels"])
    assert orc.n_iter == int(z[f"{name}_iters"])


def test_meanshift_edge_semantics():
    # SURVEY App. A.4.1 (iv): two far points -> point 0 with labels [T,F]; equal clusters -> lowest index wins
    ms = meanshift_oracle.MeanShiftOracle(0.08)
    ctr, lab = ms.fit(torch.tensor([[0., 0., 0.8], [0.5, 0., 0.8]]))
    assert lab.tolist() == [True, False] and torch.allclose(ctr, torch.tensor([0., 0., 0.8]), atol=1e-7)
    a = torch.tensor([[0., 0, 1], [0.01, 0, 1], [0.5, 0, 1], [0.51, 0, 1]])
    ctr, lab = ms.fit(a)
    assert lab.tolist() == [True, True, False, False]
    # float32 threshold: a distance equal to float32(0.08) is NOT an inlier (strict <, App. A.4.1 (ii))
    b = torch.tensor([[0., 0, 0], [float(np.float32(0.08)), 0, 0]])
    _, lab = ms.fit(b)
    assert lab.tolist() == [True, False]


def test_best_fit_transform_matches_reference(golden_dir):
    z = np.load(os.path.join(golden_dir, "bft_cases.npz"))
    for a, b, t in zip(z["A"], z["B"], z["T"]):
        assert np.array_equal(meanshift_oracle.best_fit_transform(a, b), t)
    # reference's own (weak) test: icp/test.py:24-64 -- recovered R, t within 6 sigma
    rng = np.random.default_rng(0)
    a = rng.random((10, 3))
    th = 0.3
    R = np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]])
    b = a @ R.T + np.array([0.1, -0.2, 0.3]) + rng.normal(0, 0.01, (10, 3))
    T = meanshift_oracle.best_fit_transform(a, b)
    assert np.allclose(T[:, :3], R, atol=0.06) and np.allclose(T[:, 3], [0.1, -0.2, 0.3], atol=0.06)


@pytest.mark.parametrize("case", [0, 2])
def test_frame_poses_oracle_matches_reference(golden_dir, case):
    z = np.load(os.path.join(golden_dir, "poses_ycb.npz"))
    j = case
    ids, poses, new_mask, cls_kps = frame_poses_oracle.cal_frame_poses(
        torch.from_numpy(z[f"c{j}_pcld"]), torch.from_numpy(z[f"c{j}_mask"]), torch.from_numpy(z[f"c{j}_ctr_of"]),
        torch.from_numpy(z[f"c{j}_kp_of"]), True, 22, True,
        lambda c: fixtures.get_kps(c), lambda c: fixtures.get_ctr(c), fixtures.ycb_r_lst())
    assert np.array_equal(ids, z[f"c{j}_ids"])
    assert np.array_equal(np.stack(poses), z[f"c{j}_poses"])
    assert np.array_equal(new_mask.numpy(), z[f"c{j}_new_mask"])


def test_frame_poses_lm_oracle_matches_reference(golden_dir):
    z = np.load(os.path.join(golden_dir, "poses_lm.npz"))
    for j in range(int(z["n_cases"])):
        obj = int(z[f"c{j}_obj_id"])
        poses, _ = frame_poses_oracle.cal_frame_poses_lm(
            torch.from_numpy(z[f"c{j}_pcld"]), torch.from_numpy(z[f"c{j}_mask"]), torch.from_numpy(z[f"c{j}_ctr_of"]),
            torch.from_numpy(z[f"c{j}_kp_of"]), True, 2, bool(z[f"c{j}_flt"]),
            fixtures.get_kps(obj, ds_type="linemod"), fixtures.get_ctr(obj, ds_type="linemod"))
        assert np.array_equal(poses[0], z[f"c{j}_pose"])


# ---- PointNet++ op known answers (SURVEY App. A.1-A.3) -----------------------------------------

def test_opt_n_threads_matches_reference_formula():
    # cuda_utils.h:15-19; exact for the sizes of the layer spec
    assert [pn2.opt_n_threads(n) for n in (1, 2, 3, 7, 8, 300, 512, 1024, 2048, 12288, 49152)] == \
        [1, 2, 2, 4, 8, 256, 512, 512, 512, 512, 512]


def test_fps_kat_tie_break_follows_tree_not_index():
    # All points except #0 coincide -> every candidate ties at d = 1.  Thread tid = k % 512 keeps its
    # lowest k (strict '>'); the shared-memory tree keeps the LOWER slot at each of its 9 levels, the
    # last level being (0,1) -- so even tids beat odd tids, tids = 0 mod 4 beat 2 mod 4, ...: the
    # winner is the candidate with the smallest BIT-REVERSED tid, not the smallest index.
    def cloud(n):
        xyz = np.zeros((n, 3), np.float32)
        xyz[:] = [1, 0, 2.0]
        xyz[0] = [0, 0, 2.0]
        return xyz[None]
    # n = 512: tid 0 only owns the start point (d = 0); among tids 1..511 bit-reversal is smallest
    # for tid 256 (0b100000000 -> 0b000000001)
    assert pn2.furthest_point_sampling(cloud(512), 2)[0].tolist() == [0, 256]
    # n = 1024: tid 0 also owns k = 512 (d = 1) and slot 0 wins every tie of the tree
    assert pn2.furthest_point_sampling(cloud(1024), 2)[0].tolist() == [0, 512]
    # n = 300 -> block of 256 threads (opt_n_threads): tid 0 owns k = 0 and k = 256
    assert pn2.furthest_point_sampling(cloud(300), 2)[0].tolist() == [0, 256]
    # n = 200 -> 128 threads: tid 0 owns k = 0, 128; winner k = 128
    assert pn2.furthest_point_sampling(cloud(200), 2)[0].tolist() == [0, 128]
    # n = 128 -> 128 threads, tid 0 only owns k = 0: winner is tid 64
    assert pn2.furthest_point_sampling(cloud(128), 2)[0].tolist() == [0, 64]


def test_fps_kat_skips_points_near_origin_and_spreads():
    xyz = np.array([[1, 0, 0], [0.01, 0.01, 0.01], [3, 0, 0], [2, 0, 0], [1.1, 0, 0]], np.float32)
    idx = pn2.furthest_point_sampling(xyz[None], 4)[0]
    # point 1 has |p|^2 = 3e-4 <= 1e-3 -> can never be selected (sampling_gpu.cu:100-101)
    assert idx.tolist() == [0, 2, 3, 4]


def test_ball_query_kat():
    xyz = np.array([[[0, 0, 0], [0.05, 0, 0], [1, 0, 0], [0.02, 0, 0], [0.03, 0, 0]]], np.float32)
    new = np.array([[[0, 0, 0], [5, 5, 5], [1, 0, 0]]], np.float32)
    idx = pn2.ball_query(new, xyz, 0.1, 3)[0]
    assert idx[0].tolist() == [0, 1, 3]       # first 3 hits in index order, early stop before k=4
    assert idx[1].tolist() == [0, 0, 0]       # empty ball stays zero (ball_query.cpp:19-21)
    assert idx[2].tolist() == [2, 2, 2]       # single hit pre-fills the row (ball_query_gpu.cu:34-38)
    # strict '<': a point exactly at d2 == r2 is outside
    r = np.float32(0.5)
    xyz2 = np.array([[[0, 0, 0], [float(r), 0, 0]]], np.float32)
    assert pn2.ball_query(xyz2[:, :1], xyz2, float(r), 2)[0, 0].tolist() == [0, 0]


def test_three_nn_kat():
    known = np.array([[[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 0, 0]]], np.float32)   # 1 and 3 coincide
    unk = np.array([[[0.9, 0, 0]]], np.float32)
    d, i = pn2.three_nn(unk, known)
    assert i[0, 0].tolist() == [1, 3, 0]      # ties keep the earlier index first (strict '<')
    d2, i2 = pn2.three_nn(unk, known[:, :2])  # m < 3: unused slot keeps (1e40 -> inf, 0)
    assert np.isinf(d2[0, 0, 2]) and i2[0, 0, 2] == 0


def test_group_gather_interpolate_kat():
    pts = np.arange(2 * 5, dtype=np.float32).reshape(1, 2, 5)
    idx = np.array([[[4, 0], [2, 2]]], np.int32)
    g = pn2.group_points(pts, idx)
    assert g.shape == (1, 2, 2, 2) and g[0, 1].tolist() == [[9, 5], [7, 7]]
    assert pn2.gather_points(pts, np.array([[3, 1]], np.int32))[0].tolist() == [[3, 1], [8, 6]]
    w = np.array([[[0.5, 0.25, 0.25]]], np.float32)
    out = pn2.three_interpolate(pts, np.array([[[0, 2, 4]]], np.int32), w)
    assert out[0, :, 0].tolist() == [0 * 0.5 + 2 * 0.25 + 4 * 0.25, 5 * 0.5 + 7 * 0.25 + 9 * 0.25]
    # scatter-add grads are the adjoints of the gathers
    go = np.ones((1, 2, 2, 2), np.float32)
    gg = pn2.group_points_grad(go, idx, 5)
    assert gg[0, 0].tolist() == [1, 0, 2, 0, 1]


def test_pn2_oracle_matches_reference_gpu_recording(golden_dir):
    """tests/golden/pn2_ref.npz = outputs of the UNMODIFIED reference op library (oracle/_ref/_ext.so) on a
    GPU (tests/golden/make_golden_gpu.py).  This pins the C oracle to the reference bit for bit."""
    path = os.path.join(golden_dir, "pn2_ref.npz")
    if not os.path.exists(path):
        pytest.skip("pn2_ref.npz not recorded yet")
    import importlib.util
    spec = importlib.util.spec_from_file_location("mk", os.path.join(golden_dir, "make_golden_gpu.py"))
    mk = importlib.util.module_from_spec(spec)
    sys_path = list(__import__("sys").path)
    spec.loader.exec_module(mk)
    __import__("sys").path[:] = sys_path
    z = np.load(path)
    xyz, feats = mk.inputs()
    S = mk.SPEC
    lvl = xyz
    for i, m in enumerate(S["fps_m"]):
        idx = pn2.furthest_point_sampling(lvl, m)
        assert np.array_equal(idx, z[f"fps{i}"]), f"FPS level {i}"
        nxt = np.take_along_axis(lvl, idx[..., None].astype(np.int64).repeat(3, -1), 1)
        assert np.array_equal(nxt, z[f"new_xyz{i}"])
        if i == 0:
            for j, (r, ns) in enumerate(S["bq"]):
                bq = pn2.ball_query(nxt, lvl, float(np.float32(r)), ns)
                assert np.array_equal(bq, z[f"bq{j}"]), f"ball_query {j}"
                if j == 0:
                    assert np.array_equal(pn2.group_points(feats, bq), z["group0"])
            d2, nn = pn2.three_nn(lvl, nxt)
            assert np.array_equal(nn, z["nn_idx"]) and np.array_equal(d2, z["nn_d2"])
            rng = np.random.default_rng(1)
            pf = rng.normal(size=(1, S["c_interp"], m)).astype(np.float32)
            w = rng.uniform(size=(1, S["n"], 3)).astype(np.float32)
            w /= w.sum(-1, keepdims=True)
            assert np.array_equal(pn2.three_interpolate(pf, nn, w), z["interp"])
        lvl = nxt


def test_cell_list_ball_query_prototype_matches_oracle():
    """tools/experiments/ball_cells.py (the round-2 design for the scan: voxel buckets + index-ordered hits)
    returns the reference's ball_query bit for bit -- sparse, dense (more hits than nsample), empty balls,
    duplicates, centres outside the cloud's bounding box."""
    import importlib.util
    spec = importlib.util.spec_from_file_location(
        "ball_cells", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "experiments", "ball_cells.py"))
    bc = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bc)
    rng = np.random.default_rng(11)
    for n, m, radii, nss in [(3000, 64, (0.05, 0.1), (16, 32)), (800, 40, (0.3, 0.45), (8, 16)), (500, 30, (0.01, 0.02), (4, 8))]:
        xyz = rng.uniform(-0.5, 0.5, size=(n, 3)).astype(np.float32)
        xyz[n // 2: n // 2 + 20] = xyz[:20]                                   # exact duplicates
        new = xyz[rng.choice(n, m, replace=False)].copy()
        new[0] = [2.0, 2.0, 2.0]                                              # empty ball, outside the box
        new[1] = xyz[5] + np.float32(radii[0]) * np.array([1, 0, 0], np.float32)   # a point right at the radius
        got = bc.ball_query_cells(new, xyz, radii, nss, n_buckets=256)
        for g, r, ns in zip(got, radii, nss):
            want = pn2.ball_query(new[None], xyz[None], float(np.float32(r)), ns)[0]
            assert np.array_equal(g, want), (n, r, ns)


def test_metrics_oracle_matches_reference_golden():
    """ADD / ADD-S restatement (oracle/metrics_oracle.py) against values recorded from the reference's
    Basic_Utils.cal_add_cuda / cal_adds_cuda (tests/golden/metrics.npz)"""
    import os

    import numpy as np
    import torch

    from oracle import metrics_oracle

    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "metrics.npz"))
    for i in range(len(z["which"])):
        mesh = torch.from_numpy(z["sym"] if z["which"][i] else z["mesh"])
        a = metrics_oracle.cal_add(torch.from_numpy(z["pred"][i]), torch.from_numpy(z["gt"][i]), mesh)
        s = metrics_oracle.cal_adds(torch.from_numpy(z["pred"][i]), torch.from_numpy(z["gt"][i]), mesh)
        assert np.float32(a) == z["add"][i] and np.float32(s) == z["adds"][i]
