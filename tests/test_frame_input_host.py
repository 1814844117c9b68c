"""The float64 reference of the frame-input contracts (tests/normals_ref.py) on its own, and the C ABI's
refusals of csrc/normals.cu before any launch.  No GPU needed."""
import ctypes

import numpy as np
import pytest

import normals_ref as nr
from frame_input_cases import tie_cloud
from oracle import depth_icp_oracle as dio
from pvn3d_b200 import _lib, synth


def _angle(a, b):
    """angle between rows of a and b (unsigned: the sign is checked separately)"""
    a, b = np.broadcast_arrays(np.asarray(a, np.float64), np.asarray(b, np.float64))
    return np.arctan2(np.linalg.norm(np.cross(a, b), axis=1), np.abs((a * b).sum(1)))


# ---- the sampling key and rule -----------------------------------------------------------------------------------
def test_mix64_matches_python_integers():
    rng = np.random.default_rng(0)
    z = rng.integers(0, 1 << 63, size=64, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    got = nr.mix64(z)
    assert [int(g) for g in got] == [nr.mix64_int(int(v)) for v in z]
    keys = nr.sample_keys(12345, 3, 100)
    m = (1 << 64) - 1
    base = nr.mix64_int(12345 + 4 * 0x9E3779B97F4A7C15)
    assert [int(k) for k in keys] == [nr.mix64_int((base + p) & m) for p in range(100)]


def test_keys_of_a_frame_are_distinct():
    for seed, b in ((0, 0), (2**64 - 1, 7), (99, 31)):
        k = nr.sample_keys(seed, b, 480 * 640)
        assert len(np.unique(k)) == len(k)


@pytest.mark.parametrize("nv", [399, 400, 1000, 1001, 3000])
def test_sampling_rule(nv):
    n, hw = 1000, 4096
    rng = np.random.default_rng(nv)
    valid = np.zeros(hw, bool)
    valid[rng.choice(hw, size=nv, replace=False)] = True
    idx = np.nonzero(valid)[0]
    choose, ok = nr.sample_frame(valid, n, seed=7, b=2)
    assert choose.shape == (n,) and choose.dtype == np.int64
    if nv < 400:
        assert ok == 0 and not choose.any()
        return
    assert ok == 1
    if nv <= n:                                   # np.pad(..., 'wrap')
        assert np.array_equal(choose, np.resize(idx, n))
        return
    assert np.all(np.diff(choose) > 0) and valid[choose].all()
    keys = nr.sample_keys(7, 2, hw)
    thresh = np.sort(keys[idx])[n - 1]
    assert np.array_equal(choose, idx[keys[idx] <= thresh])
    other, _ = nr.sample_frame(valid, n, seed=8, b=2)
    assert not np.array_equal(choose, other)       # the seed changes the subset
    other, _ = nr.sample_frame(valid, n, seed=7, b=3)
    assert not np.array_equal(choose, other)       # and so does the frame index


# ---- the neighbour sets ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(3))
def test_knn_matches_brute_force_with_ties_and_duplicates(seed):
    pts = tie_cloud(seed)
    got = nr.knn(pts, pts)
    want = nr.knn_brute(pts, pts)
    assert np.array_equal(got, want)
    d2 = nr.sqdist(pts[:, None], pts[want])
    assert np.all(np.diff(d2, axis=1) >= 0)
    assert (d2[:, 0] == 0).all()                                   # the query is its own neighbour
    first = want[:, 0]
    assert np.array_equal(pts[first], pts)                         # ... or an earlier duplicate of itself
    assert np.all(first <= np.arange(len(pts)))


def test_knn_respects_validity_and_non_finite_points():
    pts = tie_cloud(5)
    valid = np.random.default_rng(1).random(len(pts)) < 0.7
    pts[3] = np.nan
    q = pts[:40].copy()
    got = nr.knn(pts, q, valid)
    assert np.array_equal(got, nr.knn_brute(pts, q, valid))
    assert (got[3] == -1).all()
    assert valid[got[got >= 0]].all() and not (got == 3).any()
    assert (nr.knn(pts[:49], pts[:5]) == -1).all()                # fewer than 50 points: no neighbourhood


# ---- normals on scenes with known surfaces -----------------------------------------------------------------------
class _NoNoise:
    def normal(self, loc, scale, size):
        return np.zeros(size)


def test_normals_of_plane_and_spheres():
    K = synth.K_LINEMOD
    centres = [np.array([-0.08, 0.02, 0.7]), np.array([0.1, -0.03, 0.9])]
    radii = [0.06, 0.09]
    depth, inst = synth._render(K, centres, radii, _NoNoise())
    cloud, valid = dio.dpt_2_cld(depth, np.float32(1.0), K.astype(np.float32))
    inst = inst.ravel()
    choose, ok = nr.sample_frame(valid, 12288, seed=3, b=0)
    assert ok
    q = cloud[choose]
    idx = nr.knn(cloud, q, valid)
    n, C, lam, curv = nr.normals(cloud, idx, q)
    assert np.allclose(np.linalg.norm(n, axis=1), 1.0)
    assert ((n * q.astype(np.float64)).sum(1) <= 0).all()         # turned towards the camera
    same = (inst[idx] == inst[choose][:, None]).all(1)
    plane = same & (inst[choose] == 0)
    assert plane.sum() > 1000
    assert np.abs(n[plane] - [0.0, 0.0, -1.0]).max() < 1e-12 and (curv[plane] < 1e-12).all()
    for s, (c, r) in enumerate(zip(centres, radii)):
        sel = same & (inst[choose] == s + 1)
        true = (q[sel].astype(np.float64) - c) / r
        facing = -(true * q[sel]).sum(1) / np.linalg.norm(q[sel], axis=1) > 0.3   # away from the rim
        assert facing.sum() > 100
        ang = _angle(n[sel][facing], true[facing])
        assert np.median(ang) < 5e-3 and np.percentile(ang, 99) < 0.03


def test_normals_of_boxes_with_holes():
    d = synth.make_icp_depth_batch(1, seed=11, noise=0.0)
    cloud, valid = dio.dpt_2_cld(d["depth"][0], d["cam_scale"][0], d["K"][0])
    lab = d["label"][0].ravel()
    assert (~valid).sum() > 0.02 * valid.size                       # holes
    choose, ok = nr.sample_frame(valid, 4096, seed=5, b=0)
    q = cloud[choose]
    idx = nr.knn(cloud, q, valid)
    n, C, lam, curv = nr.normals(cloud, idx, q)
    same = (lab[idx] == lab[choose][:, None]).all(1)
    bg = same & (lab[choose] == 0)
    assert _angle(n[bg], np.array([[0.0, 0.0, -1.0]])).max() < 0.02
    boxes = same & (lab[choose] > 0)
    faces = np.einsum("qij,jk->qik", d["gt"][0][lab[choose][boxes], :, :3],
                      np.concatenate([np.eye(3), -np.eye(3)], 1))    # [q,3,6] the box's face normals
    best = np.abs(np.einsum("qi,qik->qk", n[boxes], faces)).max(1)
    ang = np.arccos(np.clip(best, 0, 1))
    assert boxes.sum() > 500 and np.median(ang) < 0.01 and np.percentile(ang, 90) < 0.05


def test_coincident_neighbourhood_gives_zero_normal():
    pts = np.concatenate([np.full((60, 3), 0.5, np.float32), np.random.default_rng(0).random((100, 3), np.float32)])
    idx = nr.knn(pts, pts[:3])
    n, C, lam, curv = nr.normals(pts, idx, pts[:3])
    assert not n.any() and not curv.any()


# ---- the ABI refuses what it cannot index before launching anything ---------------------------------------------
def _fake(i=1):
    return ctypes.c_void_p(256 * i)           # never dereferenced: every call below returns before a launch


def test_workspace_queries_refuse_int32_overflow():
    lib = _lib.load()
    assert lib.pvn3d_frame_sample_workspace_bytes(16, 480 * 640, 12288) > 0
    assert lib.pvn3d_frame_sample_workspace_bytes(7000, 480 * 640, 12288) == 0
    assert lib.pvn3d_frame_sample_workspace_bytes(0, 480 * 640, 12288) == 0
    assert lib.pvn3d_knn_normals_workspace_bytes(16, 480 * 640, 12288) > 16 * 480 * 640 * 16
    assert lib.pvn3d_knn_normals_workspace_bytes(4000, 480 * 640, 12288) == 0
    assert lib.pvn3d_knn_normals_workspace_bytes(1, 2**30, 10) == 0
    assert lib.pvn3d_knn_normals_workspace_bytes(16, 1000, 2**23) == 0


def test_entry_points_refuse_before_launch():
    lib = _lib.load()
    big = 1 << 40
    f = _fake
    # pvn3d_frame_sample: B*hw >= 2^31 -> unsupported; missing pointers / bad stride -> invalid
    assert lib.pvn3d_frame_sample(f(1), f(2), f(3), 1, None, 7000, 480 * 640, 12288, 0, f(4), 9, f(5), f(6), None,
                                  f(7), f(8), big, None) == -2
    assert lib.pvn3d_frame_sample(f(1), f(2), f(3), 1, None, 2, 480 * 640, 12288, 0, f(4), 5, f(5), f(6), None,
                                  f(7), f(8), big, None) == -1
    assert lib.pvn3d_frame_sample(None, f(2), f(3), 1, None, 2, 480 * 640, 12288, 0, f(4), 9, f(5), f(6), None,
                                  f(7), f(8), big, None) == -1
    assert lib.pvn3d_frame_sample(f(1), f(2), f(3), 1, None, 2, 480 * 640, 12288, 0, f(4), 9, f(5), f(6), f(9),
                                  f(7), f(8), big, None) == -1          # labels without a label image
    assert lib.pvn3d_frame_sample(f(1), f(2), f(3), 1, None, 2, 480 * 640, 12288, 0, f(4), 9, f(5), f(6), None,
                                  f(7), f(8), 16, None) == -4          # workspace too small
    # pvn3d_knn_normals
    assert lib.pvn3d_knn_normals(f(1), None, 480 * 640, f(2), 12288, 4000, None, f(3), 9, None, None, None, f(4), big,
                                 None) == -2
    assert lib.pvn3d_knn_normals(f(1), None, 1000, f(2), 2**23, 16, None, f(3), 9, None, None, None, f(4), big,
                                 None) == -2
    assert lib.pvn3d_knn_normals(f(1), None, 1000, f(2), 100, 2, None, f(3), 2, None, None, None, f(4), big,
                                 None) == -1
    assert lib.pvn3d_knn_normals(f(1), None, 1000, f(2), 100, 2, None, f(3), 9, None, None, None, f(4), 16,
                                 None) == -4
