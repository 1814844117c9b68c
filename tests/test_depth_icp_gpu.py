"""Full-resolution ICP scene on the GPU (csrc/icp.cu): depth back-projection bit-exact against the
reference goldens and the oracle, the nearest-neighbour label fill against a float64 brute force on
every pixel (ties, duplicates, far pixels, empty and one-point frames), and DepthIcpRefiner against the
oracle pipeline, against IcpRefiner on the same pixel cloud, and against eval_icp's recorded fits."""
import hashlib
import os

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from oracle import depth_icp_oracle as dio
from oracle import icp_oracle
from pvn3d_b200 import fixtures, synth
from pvn3d_b200.icp import DepthIcpRefiner, IcpRefiner, depth_to_cloud, dpt_2_cld, fill_label

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "depth_icp_cases.npz")
N_CLS = fixtures.YCB_N_CLASSES


@pytest.fixture(scope="module")
def z():
    return np.load(GOLDEN)


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def brute_fill(cloud, valid, pcld, point_labels, chunk=4096):
    """float64 brute force on the GPU, one op per step (nothing contracts), first index of the minimum"""
    b, p, _ = cloud.shape
    idx = torch.full((b, p), -1, dtype=torch.int64, device=cloud.device)
    for f in range(b):
        pts = pcld[f].double()
        for s in range(0, p, chunk):
            q = cloud[f, s:s + chunk].double()
            dx = torch.sub(q[:, None, 0], pts[None, :, 0])
            dy = torch.sub(q[:, None, 1], pts[None, :, 1])
            dz = torch.sub(q[:, None, 2], pts[None, :, 2])
            d2 = torch.add(torch.add(torch.mul(dx, dx), torch.mul(dy, dy)), torch.mul(dz, dz))
            idx[f, s:s + chunk] = torch.where(valid[f, s:s + chunk].bool(), torch.argmin(d2, 1), -1)
    lab = torch.where(idx >= 0, torch.gather(point_labels.long(), 1, idx.clamp(min=0)), 0)
    return lab.int(), idx.int()


def _check_fill(cloud, valid, pcld, point_labels):
    nn = torch.empty(valid.shape, dtype=torch.int32, device=cloud.device)
    got = fill_label(cloud, valid, pcld, point_labels, nn_idx=nn)
    want, widx = brute_fill(cloud, valid, pcld, point_labels)
    assert torch.equal(nn, widx)
    assert torch.equal(got, want)


@pytest.mark.parametrize("k", range(3))
def test_depth_to_cloud_matches_reference(cuda_dev, z, k):
    p = f"bp{k}_"
    dpt, cs, K = z[p + "dpt"], z[p + "cam_scale"], z[p + "K"]
    cloud, valid = depth_to_cloud(_t(dpt[None], cuda_dev), _t(K[None], cuda_dev), _t(np.array([cs]), cuda_dev))
    c, v = cloud[0].cpu().numpy(), valid[0].cpu().numpy().astype(bool)
    oc, ov = dio.dpt_2_cld(dpt, cs, K)
    assert np.array_equal(v, ov) and np.array_equal(c.view(np.uint32), oc.view(np.uint32))
    assert np.array_equal(np.nonzero(v)[0], z[p + "choose"])
    assert np.array_equal(c[v].view(np.uint32), z[p + "cld"].view(np.uint32))
    cld, choose = dpt_2_cld(dpt, cs, K, device=cuda_dev)               # the one-frame drop-in
    assert cld.dtype == np.float32 and choose.dtype == np.uint32
    assert np.array_equal(cld.view(np.uint32), z[p + "cld"].view(np.uint32)) and np.array_equal(choose, z[p + "choose"])


def test_depth_to_cloud_full_frames(cuda_dev, z):
    d = synth.make_icp_depth_batch(3, seed=4)
    d["depth"][2] = 0.0                                                 # a frame without depth
    d["depth"] = np.concatenate([d["depth"], z["full_dpt"][None]])
    d["K"] = np.concatenate([d["K"], z["full_K"][None]])
    d["K"][1] *= np.array([[1.01], [0.99], [1.0]], np.float32)        # per-frame intrinsics
    d["cam_scale"] = np.concatenate([d["cam_scale"], [z["full_cam_scale"]]]).astype(np.float32)
    cloud, valid = depth_to_cloud(_t(d["depth"], cuda_dev), _t(d["K"], cuda_dev), _t(d["cam_scale"], cuda_dev))
    cloud, valid = cloud.cpu().numpy(), valid.cpu().numpy().astype(bool)
    for f in range(4):
        oc, ov = dio.dpt_2_cld(d["depth"][f], d["cam_scale"][f], d["K"][f])
        assert np.array_equal(valid[f], ov) and np.array_equal(cloud[f].view(np.uint32), oc.view(np.uint32))
    assert not valid[2].any()
    h = hashlib.sha256()
    h.update(np.ascontiguousarray(cloud[3][valid[3]]).tobytes())
    h.update(np.nonzero(valid[3])[0].astype(np.uint32).tobytes())
    assert h.hexdigest() == str(z["full_sha"])
    assert dpt_2_cld(np.zeros((4, 5), np.float32), 1.0, np.eye(3), device=cuda_dev) == (None, None)


def test_fill_full_frames_equal_brute_force(cuda_dev):
    d = synth.make_icp_depth_batch(3, seed=6)
    dep, K, cs = _t(d["depth"], cuda_dev), _t(d["K"], cuda_dev), _t(d["cam_scale"], cuda_dev)
    cloud, valid = depth_to_cloud(dep, K, cs)
    _check_fill(cloud, valid, _t(d["pcld"], cuda_dev), _t(d["labels"], cuda_dev))


def test_fill_golden_matches_sklearn(cuda_dev, z):
    for k in range(2):
        p = f"fill{k}_"
        q, pcld, lab, tied = z[p + "cloud"], z[p + "pcld"], z[p + "point_labels"], z[p + "tied"]
        cloud, valid = _t(q[None], cuda_dev), torch.ones((1, len(q)), dtype=torch.uint8, device=cuda_dev)
        nn = torch.empty((1, len(q)), dtype=torch.int32, device=cuda_dev)
        got = fill_label(cloud, valid, _t(pcld[None], cuda_dev), _t(lab[None], cuda_dev), nn_idx=nn)
        got, nn = got[0].cpu().numpy(), nn[0].cpu().numpy()
        assert np.array_equal(nn[~tied], z[p + "index"][~tied]) and np.array_equal(got[~tied], z[p + "labels"][~tied])
        d2 = dio.sqdist64(q[tied], pcld)
        assert np.all(d2[np.arange(int(tied.sum())), nn[tied]] == d2.min(1))
        _check_fill(cloud, valid, _t(pcld[None], cuda_dev), _t(lab[None], cuda_dev))
    # the 480x640 frame: sklearn's filled mask on every pixel with an untied nearest point
    cloud, valid = depth_to_cloud(_t(z["full_dpt"][None], cuda_dev), _t(z["full_K"][None], cuda_dev),
                                  _t(np.array([z["full_cam_scale"]]), cuda_dev))
    got = fill_label(cloud, valid, _t(z["full_pcld"][None], cuda_dev), _t(z["full_point_labels"][None], cuda_dev))
    mism = int((got[0].cpu().numpy() != z["full_fill"].reshape(-1)).sum())
    assert mism <= int(z["full_fill_tied"])


def test_fill_adversarial(cuda_dev):
    rng = np.random.default_rng(12)
    s6 = 2.0 ** -6
    p, n = 40000, 600
    pts = rng.integers(-8, 8, (4, n, 3)) * s6
    pts[0, 300:] = pts[0, :300]                                               # duplicate points
    pts[3] = rng.uniform(-0.5, 0.5, (n, 3))
    q = rng.integers(-12, 12, (4, p, 3)) * s6 + np.where(rng.random((4, p, 1)) < 0.3, s6 / 2, 0.0)  # exact ties
    q[1, :1000] = rng.normal(size=(1000, 3)) * 50.0 + 100.0                  # far outside the points' box
    q[3] = rng.uniform(-0.5, 0.5, (p, 3))
    valid = (rng.random((4, p)) > 0.1).astype(np.uint8)
    valid[2] = 0                                                              # a frame with no valid pixel
    lab = rng.integers(0, N_CLS, (4, n)).astype(np.int32)
    _check_fill(_t(q.astype(np.float32), cuda_dev), _t(valid, cuda_dev), _t(pts.astype(np.float32), cuda_dev),
                _t(lab, cuda_dev))
    # one sampled point per frame
    _check_fill(_t(q.astype(np.float32), cuda_dev), _t(valid, cuda_dev), _t(pts[:, :1].astype(np.float32), cuda_dev),
                _t(lab[:, :1], cuda_dev))


@pytest.fixture(scope="module")
def depth_batch():
    return synth.make_icp_depth_batch(16, seed=17)


def _inputs(d, dev):
    return {k: _t(d[k], dev) for k in ("depth", "K", "cam_scale", "init", "present", "pcld", "labels", "label")}


def kd_nearest(q, pts, k=4):
    k = min(k, len(pts))
    _, cand = cKDTree(pts).query(q, k=k)
    cand = cand.reshape(len(q), k)
    d2 = ((q[:, None, :] - pts[cand]) ** 2).sum(-1)
    best = d2.min(1, keepdims=True)
    return np.sqrt(best[:, 0]), np.where(d2 == best, cand, np.iinfo(np.int64).max).min(1)


def test_refiner_matches_oracle_pipeline(cuda_dev, depth_batch):
    d = depth_batch
    t = _inputs(d, cuda_dev)
    ref = DepthIcpRefiner(d["models"], N_CLS, 16, device=cuda_dev)
    poses, iters, err, refined = ref.refine(t["depth"], t["K"], t["cam_scale"], t["init"], t["present"],
                                            pcld=t["pcld"], point_labels=t["labels"])
    want, _ = brute_fill(ref.cloud, ref.valid, t["pcld"], t["labels"])
    assert torch.equal(ref.labels, want)
    poses, iters, err, refined = (x.cpu().numpy() for x in (poses, iters, err, refined))
    cpts, kept_rows = ref.cluster_pts.cpu().numpy(), ref.kept_points().cpu().numpy()
    cloud, labels = ref.cloud.cpu().numpy(), ref.labels.cpu().numpy()
    n_fit = n_skip = 0
    for b in range(16):
        start = 0
        for c in range(1, N_CLS):
            cnt = int((labels[b] == c).sum())
            if not d["present"][b, c]:
                assert refined[b, c] == 0 and cpts[b, c] == 0
                start += cnt
                continue
            init = np.eye(4)
            init[:3] = d["init"][b, c].astype(np.float64)
            o = dio.object_fit(d["models"][c], cloud[b], labels[b], c, init, 2000, 1500, nn=kd_nearest)
            if o is None:
                assert refined[b, c] == 0 and cpts[b, c] == 0 and np.array_equal(poses[b, c], init[:3])
                n_skip += 1
            else:
                T, dist, i, kept = o
                assert refined[b, c] == 1 and cpts[b, c] == len(kept) and iters[b, c] == i, (b, c)
                assert np.array_equal(kept_rows[b, start:start + len(kept)], kept)
                assert np.abs(poses[b, c] - T[:3]).max() <= 1e-9 and abs(err[b, c] - dist.mean()) <= 1e-9
                n_fit += 1
            start += cnt
    assert n_fit + n_skip == 80 and n_fit >= 60


def test_refiner_equals_icp_refiner_on_the_pixel_cloud(cuda_dev, depth_batch):
    d = depth_batch
    t = _inputs(d, cuda_dev)
    ref = DepthIcpRefiner(d["models"], N_CLS, 16, device=cuda_dev)
    got = [x.clone() for x in ref.refine(t["depth"], t["K"], t["cam_scale"], t["init"], t["present"],
                                         pcld=t["pcld"], point_labels=t["labels"])]
    plain = IcpRefiner(d["models"], N_CLS, 16, 480 * 640, max_pts=2000, min_pts=1500, cluster_bandwidth=0.06,
                       device=cuda_dev)
    cloud, valid = depth_to_cloud(t["depth"], t["K"], t["cam_scale"])
    labels = fill_label(cloud, valid, t["pcld"], t["labels"])
    want = plain.refine(cloud, labels, t["init"], t["present"])
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    assert torch.equal(ref.cluster_pts, plain.cluster_pts)
    # the ground-truth label image: invalid pixels carry class 0
    got = [x.clone() for x in ref.refine(t["depth"], t["K"], t["cam_scale"], t["init"], t["present"],
                                         label_image=t["label"])]
    want = plain.refine(cloud, (t["label"].reshape(16, -1) * valid).int(), t["init"], t["present"])
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    assert torch.equal(ref.labels, (t["label"].reshape(16, -1) * valid).int())


def test_refiner_reproduces_eval_icp(cuda_dev, z):
    models = synth._box_models(N_CLS, 3000, np.random.default_rng(31))[1]
    ref = DepthIcpRefiner(models, N_CLS, 1, device=cuda_dev)
    present = _t(z["full_present"][None], cuda_dev)
    poses, iters, err, refined = ref.refine(
        _t(z["full_dpt"][None], cuda_dev), _t(z["full_K"][None], cuda_dev), _t(np.array([z["full_cam_scale"]]), cuda_dev),
        _t(z["full_init"][None], cuda_dev), present, pcld=_t(z["full_pcld"][None], cuda_dev),
        point_labels=_t(z["full_point_labels"][None], cuda_dev))
    labels = ref.labels[0].cpu().numpy()
    kept_row = ref.kept_points()[0].cpu().numpy()
    for e in range(int(z["e2e_n"])):
        p = f"e2e{e}_"
        c = int(z[p + "cls"])
        assert int(refined[0, c]) == 1 and int(iters[0, c]) == int(z[p + "i"])
        start = int(((labels >= 1) & (labels < c)).sum())
        kept = z[p + "kept"]
        assert int(ref.cluster_pts[0, c]) == len(kept) and np.array_equal(kept_row[start:start + len(kept)], kept)
        assert np.abs(poses[0, c].cpu().numpy() - z[p + "T"][:3]).max() <= 1e-9


def test_no_host_sync_and_deterministic(cuda_dev):
    d = synth.make_icp_depth_batch(3, seed=9)
    t = _inputs(d, cuda_dev)
    ref = DepthIcpRefiner(d["models"], N_CLS, 4, device=cuda_dev)
    args = (t["depth"], t["K"], t["cam_scale"], t["init"], t["present"])
    first = [x.clone() for x in ref.refine(*args, pcld=t["pcld"], point_labels=t["labels"])]
    first_labels, first_pts = ref.labels[:3].clone(), ref.cluster_pts[:3].clone()
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        again = ref.refine(*args, pcld=t["pcld"], point_labels=t["labels"])
        ref.refine(*args, label_image=t["label"])
        again = [x.clone() for x in ref.refine(*args, pcld=t["pcld"], point_labels=t["labels"])]
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    torch.cuda.synchronize()
    for a, b in zip(first, again):
        assert torch.equal(a, b)
    assert torch.equal(first_labels, ref.labels[:3]) and torch.equal(first_pts, ref.cluster_pts[:3])
    assert first[3].any()
