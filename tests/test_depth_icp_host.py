"""Full-resolution ICP scene, host side (no GPU): the oracle against the goldens recorded from the
reference's dpt_2_cld, sklearn's NearestNeighbors and eval_icp's per-object pipeline; the C-ABI binding
table and header; argument checks that launch nothing; the depth-batch generator."""
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import depth_icp_oracle as dio
from pvn3d_b200 import _lib, icp, synth

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "depth_icp_cases.npz")
HEADER = os.path.join(os.path.dirname(HERE), "include", "pvn3d_b200.h")
NAMES = ("pvn3d_depth_to_cloud", "pvn3d_label_fill_workspace_bytes", "pvn3d_label_fill")


@pytest.fixture(scope="module")
def z():
    return np.load(GOLDEN)


def test_goldens_cover_the_documented_cases(z):
    assert os.path.getsize(GOLDEN) < 2 << 20
    assert len(z["bp_names"]) == 3 and len(z["fill_names"]) == 2
    assert z["full_dpt"].shape == (480, 640) and (z["full_dpt"] == 0).any()          # holes
    assert z["fill1_tied"].sum() > 100                                                  # exact ties exercised
    assert int(z["e2e_n"]) == 2


@pytest.mark.parametrize("k", range(3))
def test_oracle_back_projection_is_the_reference(z, k):
    p = f"bp{k}_"
    cloud, valid = dio.dpt_2_cld(z[p + "dpt"], z[p + "cam_scale"], z[p + "K"])
    assert np.array_equal(np.nonzero(valid)[0], z[p + "choose"])
    assert np.array_equal(cloud[valid].view(np.uint32), z[p + "cld"].view(np.uint32))
    assert not cloud[~valid].any()


def test_oracle_back_projection_full_frame(z):
    cloud, valid = dio.dpt_2_cld(z["full_dpt"], z["full_cam_scale"], z["full_K"])
    h = hashlib.sha256()
    h.update(np.ascontiguousarray(cloud[valid]).tobytes())
    h.update(np.nonzero(valid)[0].astype(np.uint32).tobytes())
    assert h.hexdigest() == str(z["full_sha"])


@pytest.mark.parametrize("k", range(2))
def test_oracle_fill_is_sklearn(z, k):
    p = f"fill{k}_"
    q, pcld, lab = z[p + "cloud"], z[p + "pcld"], z[p + "point_labels"]
    labels, idx = dio.fill_label(q, np.ones(len(q), bool), pcld, lab)
    tied = z[p + "tied"]
    assert np.array_equal(idx[~tied], z[p + "index"][~tied])
    assert np.array_equal(labels[~tied], z[p + "labels"][~tied])
    d2 = dio.sqdist64(q[tied], pcld)                   # sklearn's pick is one of the tied points
    best = d2.min(1)
    assert np.all(d2[np.arange(len(best)), z[p + "index"][tied]] == best)
    assert np.all(d2[np.arange(len(best)), idx[tied]] == best)


def test_oracle_fill_lowest_index_and_invalid():
    pcld = np.array([[0, 0, 0], [1, 0, 0], [0, 0, 0], [1, 0, 0]], np.float32)
    cloud = np.array([[0.5, 0, 0], [2, 0, 0], [-1, 0, 0], [9, 9, 9]], np.float32)
    labels, idx = dio.fill_label(cloud, np.array([1, 1, 1, 0], bool), pcld, np.array([5, 6, 7, 8], np.int32))
    assert idx.tolist() == [0, 1, 0, -1] and labels.tolist() == [5, 6, 5, 0]


def test_oracle_pipeline_is_eval_icp(z):
    cloud, valid = dio.dpt_2_cld(z["full_dpt"], z["full_cam_scale"], z["full_K"])
    labels = z["full_fill"].reshape(-1).astype(np.int32)            # sklearn's fill (0 on invalid pixels)
    assert not labels[~valid].any()
    # the frame is make_icp_depth_batch(1, seed=31)'s; its models are the first draws of that seed
    models = synth._box_models(len(z["full_present"]), 3000, np.random.default_rng(31))[1]
    for e in range(int(z["e2e_n"])):
        p = f"e2e{e}_"
        c = int(z[p + "cls"])
        init = np.eye(4)
        init[:3] = z["full_init"][c].astype(np.float64)
        T, d, i, kept = dio.object_fit(models[c], cloud, labels, c, init, 2000, 1500, 0.06, 500, 1e-9)
        assert i == int(z[p + "i"]) and np.array_equal(kept, z[p + "kept"])
        assert np.abs(T - z[p + "T"]).max() <= 1e-12 and abs(d.mean() - float(z[p + "err"])) <= 1e-12


def test_symbols_in_binding_table_and_header():
    header = open(HEADER).read()
    for name in NAMES:
        assert name in _lib._SIGNATURES and f"{name}(" in header


def _lib_or_skip():
    try:
        return _lib.load()
    except _lib.Pvn3dError:
        pytest.skip("kernel library not built")


def test_argument_checks_launch_nothing():
    lib = _lib_or_skip()
    bad = 0x1000                 # never dereferenced: every call below must return before any launch
    ws = (bad & ~255) + 256
    before = lib.pvn3d_launch_count()
    d2c = lambda b, h, w, cloud=bad: lib.pvn3d_depth_to_cloud(bad, bad, bad, b, h, w, cloud, bad, 0)
    assert d2c(0, 480, 640) == -1 and d2c(1, 0, 640) == -1 and d2c(1, 480, -1) == -1
    assert d2c(1, 480, 640, cloud=0) == -1
    assert d2c(6991, 480, 640) == -2                                 # 6991*480*640 >= 2^31
    assert d2c(1, 46341, 46341) == -2
    assert lib.pvn3d_label_fill_workspace_bytes(16, 12288) > 0
    assert lib.pvn3d_label_fill_workspace_bytes(0, 12288) == 0
    assert lib.pvn3d_label_fill_workspace_bytes(16, 0) == 0
    assert lib.pvn3d_label_fill_workspace_bytes(65536, 10) == 0
    assert lib.pvn3d_label_fill_workspace_bytes(2, 1 << 30) == 0
    need = lib.pvn3d_label_fill_workspace_bytes(16, 12288)
    fill = lambda hw, b, n, ws_=ws, nbytes=1 << 40, out=bad: lib.pvn3d_label_fill(
        bad, bad, hw, bad, bad, b, n, out, 0, ws_, nbytes, 0)
    assert fill(307200, 6991, 12288) == -2                           # B*H*W >= 2^31
    assert fill(307200, 16, 12288, nbytes=need - 1) == -4
    assert fill(307200, 16, 12288, ws_=ws + 16) == -1                # workspace not 256-B aligned
    assert fill(307200, 16, 12288, out=0) == -1
    assert fill(0, 16, 12288) == -1 and fill(307200, 16, 0) == -1 and fill(307200, 0, 12288) == -1
    assert lib.pvn3d_launch_count() == before


def test_python_argument_checks():
    dep = torch.zeros(2, 4, 5)
    with pytest.raises(ValueError, match="K"):
        icp.depth_to_cloud(dep, torch.zeros(2, 3, 4), torch.ones(2))
    with pytest.raises(ValueError, match="CUDA"):
        icp.depth_to_cloud(dep, torch.zeros(2, 3, 3), torch.ones(2))              # CPU tensors
    with pytest.raises(ValueError, match="shapes"):
        icp.fill_label(torch.zeros(2, 20, 3), torch.zeros(2, 19, dtype=torch.uint8), torch.zeros(2, 7, 3),
                       torch.zeros(2, 7, dtype=torch.int32))
    with pytest.raises(ValueError, match="CUDA"):
        icp.fill_label(torch.zeros(2, 20, 3), torch.zeros(2, 20, dtype=torch.uint8), torch.zeros(2, 7, 3),
                       torch.zeros(2, 7, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="CUDA only"):
        icp.DepthIcpRefiner({1: np.zeros((4, 3))}, 2, 1, device="cpu")
    with pytest.raises(RuntimeError, match="CUDA only"):
        icp.dpt_2_cld(np.zeros((4, 5), np.float32), 1.0, np.eye(3), device="cpu")
    with pytest.raises(ValueError, match="64-bit"):
        icp.DepthIcpRefiner({1: np.zeros((4, 3))}, 2, 6991, device="cuda:0")


def _digest(d, keys):
    h = hashlib.sha256()
    for k in keys:
        h.update(np.ascontiguousarray(d[k]).tobytes())
    return h.hexdigest()


def test_depth_batch_generator():
    keys = ("depth", "K", "cam_scale", "label", "gt", "init", "present", "pcld", "labels", "choose")
    a = synth.make_icp_depth_batch(2, seed=5, height=120, width=160, n_sample=1000)
    b = synth.make_icp_depth_batch(2, seed=5, height=120, width=160, n_sample=1000)
    assert _digest(a, keys) == _digest(b, keys)                       # deterministic
    ref = synth.make_icp_batch(1, 5, 10, seed=5)                      # the same box models
    assert all(np.array_equal(m, r) for m, r in zip(a["models"][1:], ref["models"][1:]))
    assert a["depth"].shape == (2, 120, 160) and a["depth"].dtype == np.float32
    for f in range(2):
        ch = a["choose"][f]
        assert np.all(np.diff(ch) > 0) and np.all(a["depth"][f].ravel()[ch] > 0)   # raster order, valid pixels
        holes = a["depth"][f] == 0
        assert 0.01 < holes.mean() < 0.2
        flipped = a["labels"][f] != a["label"][f].ravel()[ch]
        assert 0 < flipped.sum() <= round(0.03 * 1000)
        assert set(np.unique(a["label"][f])) <= {0} | set(np.nonzero(a["present"][f])[0])   # a 120x160 crop
        cloud, valid = dio.dpt_2_cld(a["depth"][f], a["cam_scale"][f], a["K"][f])
        assert np.array_equal(cloud[ch], a["pcld"][f])                 # dpt_2_cld's arithmetic
