"""csrc/augment.cu on the GPU against the numpy restatement tests/augment_ref.py (itself checked against cv2 / PIL /
torchvision and the reference's methods by tests/golden/make_golden_augment.py): each building block exhaustively,
the whole stage with explicit records and with device draws replayed on the host, determinism, the draws'
distributions, the noise moments, graph capture and an augment -> train_batch(fill="multiscale") batch."""
import numpy as np
import pytest
import torch
from scipy import stats

import augment_ref as R
import train_ref as TR
from pvn3d_b200 import augment as A
from pvn3d_b200 import train_utils as T
from pvn3d_b200.frame_input import FrameInputBuilder

pytestmark = pytest.mark.gpu


def _all_triples():
    a = np.arange(256 ** 3, dtype=np.int64)
    return np.stack([a >> 16, (a >> 8) & 255, a & 255], -1).astype(np.uint8)


@pytest.fixture(scope="module")
def triples():
    return _all_triples()


@pytest.mark.parametrize("op,fn", [(0, R.cv_bgr2hsv), (1, R.cv_hsv2bgr), (2, R.pil_rgb2hsv), (3, R.pil_hsv2rgb),
                                   (4, R.pil_l), (7, lambda x: R.cv_hsv2bgr(x, vector=False))])
def test_colour_ops_exhaustive(cuda_dev, triples, op, fn):
    x = torch.from_numpy(triples).to(cuda_dev)
    out = torch.empty(len(triples) * (1 if op == 4 else 3), dtype=torch.uint8, device=cuda_dev)
    got = A.probe(op, x, out).cpu().numpy()
    want = fn(triples).reshape(-1)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, (op, bad[:5], got[bad[:5]], want[bad[:5]])


def test_hsv_scale_exhaustive(cuda_dev, triples):
    """the whole HSV augmentor (BGR2HSV, S/V scaling and truncation, HSV2BGR) on every colour, both datasets' ranges"""
    h, w = -(-len(triples) // 4111), 4111                       # rows of 128 vectors of 32 pixels and a tail of 15
    img = np.resize(triples, (h * w, 3)).reshape(h, w, 3)
    aug = A.FrameAugmenter(1, "ycb", h, w, device=cuda_dev)
    d = torch.from_numpy(img[None]).to(cuda_dev)
    z = torch.zeros((1, h, w), dtype=torch.float32, device=cuda_dev)
    lab = torch.ones((1, h, w), dtype=torch.uint8, device=cuda_dev)
    for s, v in ((1.25, 1.35), (1.4471, 1.1502), (0.75, 1.15), (0.9137, 0.8501)):
        p = R.blank_params(1)
        p["n_pass"] = 1
        p["passes"]["s_factor"][0, 0], p["passes"]["v_factor"][0, 0] = s, v
        got, _ = aug.apply(d, z, lab, d, lab, z, aug.from_records(p))
        want = R.hsv_scale(img, s, v)
        assert np.array_equal(got[0].permute(1, 2, 0).cpu().numpy(), want), (s, v)


def test_gaussian_taps_dense_sigma_sweep(cuda_dev):
    sig = np.concatenate([[0.0, -1.0, 1e-300, 1e-12, 1e-6], np.linspace(0, 1, 20001)[1:],
                          np.random.default_rng(3).random(5000)])
    args = np.stack([np.repeat([3.0, 5.0], len(sig)), np.tile(sig, 2)], -1)
    out = torch.empty((len(args), 5), dtype=torch.int32, device=cuda_dev)
    got = A.probe(5, torch.from_numpy(args).to(cuda_dev), out).cpu().numpy()
    for (k, s), g in zip(args, got):
        k = int(k)
        assert np.array_equal(g[:k], R.gaussian_kernel_fixed(k, s)), (k, s, g)


def test_motion_line_every_angle_and_length(cuda_dev):
    args = np.array([(a, n) for a in range(360) for n in range(1, 16)], np.int32)
    out = torch.empty((len(args), 64), dtype=torch.int32, device=cuda_dev)
    got = A.probe(6, torch.from_numpy(args).to(cuda_dev), out).cpu().numpy()
    for (a, n), g in zip(args, got):
        side, pts = R.motion_line(int(a), int(n))
        want = sorted(set(y * 256 + x for (y, x) in pts))
        assert g[0] == side and list(g[2:2 + g[1]]) == (want if side else []), (a, n)


def _inputs(rng, b, h, w, back_ch=1):
    rgb = rng.integers(0, 256, (b, h, w, 3), dtype=np.uint8)
    rgb[:, : h // 4] = 255                                   # saturated rows
    rgb[:, h // 4: h // 3] = rng.integers(0, 3, (b, h // 3 - h // 4, w, 3))
    depth = rng.integers(0, 2000, (b, h, w)).astype(np.float32)
    depth[depth < 300] = 0
    labels = (rng.random((b, h, w)) < 0.4).astype(np.uint8) * rng.integers(1, 22, (b, h, w)).astype(np.uint8)
    labels[0] = 0                                            # all background
    if b > 1:
        labels[1] = 3                                        # all foreground
    back = rng.integers(0, 256, (b, h, w, 3), dtype=np.uint8)
    bl = (rng.random((b, h, w) if back_ch == 1 else (b, h, w, 3)) < 0.3).astype(np.uint8) * 9
    bd = rng.integers(0, 3000, (b, h, w)).astype(np.float32)
    return rgb, depth, labels, back, bl, bd


def _replay(dataset, recs, ins, noise, stages_dev, rgb_dev, depth_dev):
    rgb, depth, labels, back, bl, bd = ins
    for f in range(len(recs)):
        nz = None if noise is None else noise[f]
        out, dpt, st = R.augment_frame(rgb[f], depth[f], labels[f], back[f], bl[f], bd[f], recs[f], dataset, nz)
        for i, s in enumerate(st):
            assert np.array_equal(stages_dev[f, i], s), (dataset, f, "stage", i, recs[f])
        assert np.array_equal(rgb_dev[f], out), (dataset, f)
        assert np.array_equal(depth_dev[f], dpt), (dataset, f)


def _explicit_records(dataset, rng, b):
    kinds = [R.KIND_SYN] * b if dataset == R.YCB else [R.KIND_RENDER, R.KIND_REAL, R.KIND_FUSE] * b
    p = R.host_draw(rng, dataset, kinds[:b])
    if dataset == R.YCB:                                      # frame 0 runs the second pass
        p[0]["n_pass"] = 2
        p[0]["passes"][1] = p[0]["passes"][0]
        p[0]["passes"]["s_factor"][1], p[0]["passes"]["noise_key"][1] = 1.3, 77
    # every branch at least once: sharpen, motion (incl. length 1), both blur sizes, sigma -> 0, extra noise
    for f in range(b):
        for q in range(2):
            ps = p[f]["passes"][q]
            if p[f]["n_pass"] > q:
                ps["motion"] = ps["gauss"] = 1
                ps["sharpen"] = int(dataset == R.YCB)
                ps["extra"] = int(dataset == R.YCB and f % 2 == 0)
                ps["ksize"] = 5 if (f + q) % 2 else 3
                ps["sigma"] = [0.0, 1e-7, 0.43, 0.999][(f + q) % 4]
                ps["length"] = [1, 15, 7, 2][(f + 2 * q) % 4]
    return p


@pytest.mark.parametrize("dataset,h,w,back_ch", [("ycb", 37, 53, 1), ("ycb", 5, 3, 1), ("linemod", 29, 41, 3),
                                                  ("linemod", 24, 32, 1)])
def test_stage_with_explicit_records(cuda_dev, dataset, h, w, back_ch):
    rng = np.random.default_rng(h * w)
    b = 4
    ins = _inputs(rng, b, h, w, back_ch)
    recs = _explicit_records(dataset, rng, b)
    aug = A.FrameAugmenter(b, dataset, h, w, debug=True, device=cuda_dev)
    d = [torch.from_numpy(x).to(cuda_dev) for x in ins]
    rgb_o, dep_o = aug.apply(*d, aug.from_records(recs))
    _replay(dataset, recs, ins, aug.noise.cpu().numpy(), aug.stages.cpu().numpy(), rgb_o.cpu().numpy(),
            dep_o.cpu().numpy())


@pytest.mark.parametrize("dataset", ["ycb", "linemod"])
def test_stage_with_device_draws(cuda_dev, dataset):
    rng = np.random.default_rng(7)
    h, w = 480, 640
    kinds = [1, 0, 1, 1] if dataset == "ycb" else [1, 0, 2, 1]
    b = len(kinds)
    ins = _inputs(rng, b, h, w)
    aug = A.FrameAugmenter(b, dataset, h, w, debug=True, device=cuda_dev)
    d = [torch.from_numpy(x).to(cuda_dev) for x in ins]
    seed = 1234 if dataset == "ycb" else 99
    params = aug.draw(seed, kinds)
    rgb_o, dep_o = aug.apply(*d, params)
    recs = A.records(params)
    assert recs["kind"].tolist() == kinds
    _replay(dataset, recs, ins, aug.noise.cpu().numpy(), aug.stages.cpu().numpy(), rgb_o.cpu().numpy(),
            dep_o.cpu().numpy())
    # the same seed gives the same bits; another seed other draws
    first = (params.clone(), rgb_o.clone(), dep_o.clone())
    rgb2, dep2 = aug.apply(*d, aug.draw(seed, kinds))
    assert torch.equal(aug.params[:b], first[0]) and torch.equal(rgb2, first[1]) and torch.equal(dep2, first[2])
    assert not torch.equal(aug.draw(seed + 1, kinds), first[0])


def _binom_ok(k, n, p, z=5.0):
    return abs(k - n * p) <= z * np.sqrt(n * p * (1 - p)) + 1


@pytest.mark.parametrize("dataset", ["ycb", "linemod"])
def test_draw_distributions(cuda_dev, dataset):
    n = 20000
    kinds = torch.ones(n, dtype=torch.int32, device=cuda_dev)           # syn / render: every branch is drawn
    aug = A.FrameAugmenter(n, dataset, 1, 1, device=cuda_dev)
    r = A.records(aug.draw(2024, kinds))
    assert (r["kind"] == 1).all() and (r["back"] == 1).all()
    assert (r["jitter"] == (1 if dataset == "ycb" else 0)).all()
    assert _binom_ok(int((r["n_pass"] == 2).sum()), n, 0.2) and set(np.unique(r["n_pass"])) == {1, 2}
    p1 = r["passes"][:, 0]
    lo, hi = R.S_RANGE[dataset]
    assert stats.kstest(p1["s_factor"], stats.uniform(lo, hi - lo).cdf).pvalue > 1e-4
    lo, hi = R.V_RANGE[dataset]
    assert stats.kstest(p1["v_factor"], stats.uniform(lo, hi - lo).cdf).pvalue > 1e-4
    for flag in ("motion", "gauss") + (("sharpen", "extra") if dataset == "ycb" else ()):
        assert _binom_ok(int(p1[flag].sum()), n, 0.2), flag
    assert _binom_ok(int((p1["ksize"] == 5).sum()), n, 0.2)
    assert stats.kstest(p1["sigma"], "uniform").pvalue > 1e-4
    assert p1["angle"].min() == 0 and p1["angle"].max() == 359
    assert stats.chisquare(np.bincount(p1["angle"], minlength=360)).pvalue > 1e-4
    assert stats.chisquare(np.bincount(p1["length"], minlength=16)[1:]).pvalue > 1e-4
    if dataset == "ycb":
        assert stats.kstest(p1["sharpen_w"], stats.uniform(9, 3).cdf).pvalue > 1e-4
        ns = p1["noise_sigma"]
        # randint(15) w.p. 0.8, else randint(25): P(sigma = s) = 0.8/15 + 0.2/25 below 15, 0.2/25 from 15 to 24
        pk = np.array([0.8 / 15 + 0.2 / 25] * 15 + [0.2 / 25] * 10)
        assert ns.min() >= 0 and ns.max() <= 24
        assert stats.chisquare(np.bincount(ns, minlength=25), pk * n).pvalue > 1e-4
    else:
        assert (p1["sharpen"] == 0).all() and (p1["extra"] == 0).all() and (p1["noise_sigma"] == 0).all()
    # pass 2 only where drawn
    two = r["n_pass"] == 2
    assert (r["passes"][~two, 1]["motion"] == 0).all() and (r["passes"][~two, 1]["s_factor"] == 1).all()
    # jitter (every YCB frame; LineMOD real png frames only)
    kinds = torch.zeros(n, dtype=torch.int32, device=cuda_dev)
    r = A.records(aug.draw(77, kinds))
    assert (r["jitter"] == 1).all() and (r["n_pass"] == 0).all() and (r["back"] == 0).all()
    for f in ("brightness", "contrast", "saturation"):
        assert stats.kstest(r[f], stats.uniform(0.8, 0.4).cdf).pvalue > 1e-4, f
    assert stats.kstest(r["hue"], stats.uniform(-0.05, 0.1).cdf).pvalue > 1e-4
    perms = {tuple(o) for o in r["order"].tolist()}
    assert len(perms) == 24
    codes = (r["order"] * np.array([64, 16, 4, 1])).sum(1)
    assert stats.chisquare(np.unique(codes, return_counts=True)[1]).pvalue > 1e-4
    if dataset == "linemod":
        r = A.records(aug.draw(5, torch.full((n,), 2, dtype=torch.int32, device=cuda_dev)))
        assert (r["jitter"] == 0).all() and (r["n_pass"] == 0).all() and (r["back"] == 0).all()


def test_noise_moments(cuda_dev):
    h, w = 480, 640
    aug = A.FrameAugmenter(2, "ycb", h, w, debug=True, device=cuda_dev)
    recs = R.blank_params(2)
    recs["n_pass"] = 2
    recs["passes"]["extra"] = 1
    recs["passes"]["noise_sigma"] = 3
    recs["passes"]["noise_key"] = [[11, 12], [13, 14]]
    recs["passes"]["extra_key"] = [[21, 22], [23, 24]]
    z = torch.zeros((2, h, w), dtype=torch.float32, device=cuda_dev)
    img = torch.full((2, h, w, 3), 128, dtype=torch.uint8, device=cuda_dev)
    lab = torch.ones((2, h, w), dtype=torch.uint8, device=cuda_dev)
    aug.apply(img, z, lab, img, lab, z, aug.from_records(recs))
    fields = aug.noise.cpu().numpy().astype(np.float64)
    m = fields.size
    assert abs(fields.mean()) < 5 / np.sqrt(m)
    assert abs(fields.var() - 1) < 5 * np.sqrt(2 / m)
    assert abs(stats.skew(fields.ravel())) < 5 * np.sqrt(6 / m)
    assert abs(stats.kurtosis(fields.ravel())) < 5 * np.sqrt(24 / m)
    flat = fields.reshape(8, -1)                                    # four keys x two frames: no two fields alike
    c = np.corrcoef(flat)
    assert np.abs(c - np.eye(8)).max() < 5 / np.sqrt(flat.shape[1])
    # channels of one pixel are independent too
    px = fields.reshape(-1, 3)
    assert np.abs(np.corrcoef(px.T) - np.eye(3)).max() < 5 / np.sqrt(len(px))


def test_graph_capture_and_replay(cuda_dev):
    rng = np.random.default_rng(5)
    b, h, w = 3, 96, 128
    ins = [torch.from_numpy(x).to(cuda_dev) for x in _inputs(rng, b, h, w)]
    kinds = torch.tensor([1, 0, 1], dtype=torch.int32, device=cuda_dev)
    aug = A.FrameAugmenter(b, "ycb", h, w, device=cuda_dev)
    s = torch.cuda.Stream(cuda_dev)
    s.wait_stream(torch.cuda.current_stream(cuda_dev))
    with torch.cuda.stream(s):
        aug.apply(*ins, aug.draw(8, kinds))                              # warm-up outside the capture
    torch.cuda.current_stream(cuda_dev).wait_stream(s)
    want = [t.clone() for t in aug.apply(*ins, aug.draw(8, kinds))]
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = aug.apply(*ins, aug.draw(8, kinds))
    aug.rgb_out.zero_()
    aug.depth_out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], want[0]) and torch.equal(out[1], want[1])


def test_augment_then_train_batch(cuda_dev):
    b, n, h, w = 3, 12288, 480, 640
    depth, K, cs, rgb, label, ids, rts = TR.raw_frames(b, h, w, 0, sparse=(1,))
    rng = np.random.default_rng(9)
    back = rng.integers(0, 256, (b, h, w, 3), dtype=np.uint8)
    back_lab = np.zeros((b, h, w), np.uint8)
    back_dpt = np.full((b, h, w), 8500, np.float32)
    depth[0, :50] = 0                                              # holes the composite fills from the background
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda_dev)  # noqa: E731
    aug = A.FrameAugmenter(b, "ycb", h, w, device=cuda_dev)
    builder = FrameInputBuilder(b, n, fill="multiscale", device=cuda_dev)
    targets = T.TrainTargets(device=cuda_dev)
    kinds = d(np.array([1, 1, 0], np.int32))
    ins = [d(x) for x in (rgb.transpose(0, 2, 3, 1), depth, label.astype(np.uint8), back, back_lab, back_dpt)]
    K_d, cs_d, lab_d, ids_d, rts_d = d(K), d(cs), d(label), d(ids), d(rts)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        params = aug.draw(31, kinds)
        rgb_a, dpt_a = aug.apply(*ins, params)
        out = T.train_batch(builder, targets, dpt_a, K_d, cs_d, rgb_a, lab_d, ids_d, rts_d, seed=11)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    ok = out[-1]
    # frame 1 keeps 300 valid pixels of its own, but the composite fills its background from the real frame
    assert ok.tolist() == [1, 1, 1]
    assert float(dpt_a[0, :50].min()) == 8500.0 and torch.equal(dpt_a[2], d(depth[2]))
    assert tuple(out[0].shape) == (b, 3, h, w) and bool(torch.isfinite(out[4]).all())
