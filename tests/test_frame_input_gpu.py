"""FrameInputBuilder and estimate_normals (csrc/normals.cu) against the float64 reference of
tests/normals_ref.py: the sampled pixels, ok flags and columns 0..5 of cld_rgb_nrm bit for bit, the 50
neighbour indices index for index in both normal modes, and the normals against the reference covariance.
Frames: LineMOD-shape spheres over a plane, a frame with fewer valid pixels than points (wrap duplicates),
one with fewer than 400 (not a frame), and YCB-shape box scenes with holes at 480x640."""
import numpy as np
import pytest
import torch

import normals_ref as nr
from pvn3d_b200 import network, synth, testing
from pvn3d_b200.frame_input import FrameInputBuilder, estimate_normals

pytestmark = pytest.mark.gpu

N = 12288


def angle(a, b):
    """unsigned angle between rows, from |a x b| and |a . b| (arccos of a float32 dot product near 1 would
    report the rounding of |a| as an angle of ~1e-4 rad)"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.arctan2(np.linalg.norm(np.cross(a, b), axis=1), np.abs((a * b).sum(1)))


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _linemod_batch(seed):
    """4 frames of LineMOD shape (cam_scale 1000, depth in mm as a PNG holds it): two sphere scenes, one with
    3000 valid pixels (< N: wrapped), one with 399 (ok = 0)"""
    rng = np.random.default_rng(seed)
    K = synth.K_LINEMOD.astype(np.float32)
    depth = np.zeros((4, synth.H, synth.W), np.float32)
    for b in range(4):
        centres = [np.array([rng.uniform(-0.1, 0.1), rng.uniform(-0.05, 0.05), rng.uniform(0.6, 0.9)])
                   for _ in range(2)]
        d, _ = synth._render(K.astype(np.float64), centres, [0.05, 0.08], rng)
        depth[b] = np.round(d * 1000.0)
    for b, keep in ((2, 3000), (3, 399)):
        flat = depth[b].ravel()
        drop = rng.choice(flat.size, size=flat.size - keep, replace=False)
        flat[drop] = 0.0
    rgb = rng.integers(0, 256, size=(4, 3, synth.H, synth.W), dtype=np.uint8)
    return dict(depth=depth, K=np.repeat(K[None], 4, 0), cam_scale=np.full(4, 1000.0, np.float32), rgb=rgb,
                label=(depth > 0).astype(np.int32) * 7)


def _ycb_batch(seed):
    d = synth.make_icp_depth_batch(2, seed=seed)
    rng = np.random.default_rng(seed)
    d["rgb"] = rng.uniform(0, 255, size=(2, 3, synth.H, synth.W)).astype(np.float32)
    return d


def _oracle(d, mode, seed):
    from oracle import depth_icp_oracle as dio

    clouds, valids = zip(*(dio.dpt_2_cld(d["depth"][b], d["cam_scale"][b], d["K"][b]) for b in range(len(d["depth"]))))
    cloud, valid = np.stack(clouds), np.stack(valids)
    rgb = d["rgb"].reshape(len(cloud), 3, -1)
    return nr.frame_input(cloud, valid, rgb, N, seed, mode), cloud


def _check_normals(got32, got64, want, C, lam, q, ok):
    """the normal contract on every point of the ok frames"""
    okp = np.repeat(ok.astype(bool), q.shape[1])
    got32, got64 = got32.reshape(-1, 3)[okp], got64.reshape(-1, 3)[okp]
    want, C, lam, q = want.reshape(-1, 3)[okp], C.reshape(-1, 3, 3)[okp], lam.reshape(-1, 3)[okp], \
        q.reshape(-1, 3)[okp].astype(np.float64)
    assert np.array_equal(got32, got64.astype(np.float32))
    tr = np.trace(C, axis1=1, axis2=2)
    zero = tr == 0
    assert not got64[zero].any()
    g, Cz, l0, t = got64[~zero], C[~zero], lam[~zero, 0], tr[~zero]
    assert np.allclose(np.linalg.norm(g, axis=1), 1.0, atol=1e-12)
    res = np.linalg.norm(np.einsum("qij,qj->qi", Cz, g) - l0[:, None] * g, axis=1)
    assert (res <= 1e-9 * t).all(), f"worst residual / trace {np.max(res / t):.3e}"
    sep = (lam[~zero, 1] - l0) / t >= 1e-3
    w = want[~zero]
    ang = angle(got32[~zero][sep], w[sep])
    assert ang.size == 0 or ang.max() <= 1e-6, f"worst angle {ang.max():.3e} rad"
    qq = q[~zero]
    clear = sep & (np.abs((w * qq).sum(1)) >= 1e-6 * np.linalg.norm(qq, axis=1))
    assert np.array_equal(np.sign((g[clear] * qq[clear]).sum(1)), np.sign((w[clear] * qq[clear]).sum(1)))
    return sep.mean()


def _run_and_check(d, mode, seed, dev):
    want, cloud = _oracle(d, mode, seed)
    b = len(d["depth"])
    fib = FrameInputBuilder(b, N, normals=mode, debug=True, device=dev)
    cld, rgb, choose, pcld, ok, labels = fib.build(
        _t(d["depth"], dev), _t(d["K"], dev), _t(d["cam_scale"], dev), _t(d["rgb"], dev), seed,
        label_image=_t(d["label"], dev))
    torch.cuda.synchronize()
    ok_h = ok.cpu().numpy()
    assert np.array_equal(ok_h, want["ok"])
    ch = choose.cpu().numpy()
    assert ch.shape == (b, 1, N) and np.array_equal(ch[:, 0], want["choose"])
    c = cld.cpu().numpy()
    assert np.array_equal(c[:, :, :6].view(np.uint32), want["cld6"].view(np.uint32))
    assert np.array_equal(pcld.cpu().numpy().view(np.uint32), want["cld6"][:, :, :3].view(np.uint32))
    assert torch.equal(rgb, _t(d["rgb"], dev).float())
    lab = d["label"].reshape(b, -1)
    want_lab = np.stack([np.where(want["ok"][f], lab[f][want["choose"][f]], 0) for f in range(b)])
    assert np.array_equal(labels.cpu().numpy(), want_lab)
    assert np.array_equal(fib.nn_idx.cpu().numpy().astype(np.int64), want["idx"])
    assert not c[ok_h == 0].any()
    frac = _check_normals(c[:, :, 6:], fib.normals64.cpu().numpy(), want["n"], want["C"], want["lam"],
                          want["cld6"][:, :, :3], ok_h)
    assert frac > 0.5                   # the angle and sign checks cover most points
    return fib


@pytest.mark.parametrize("mode", ["sampled", "full"])
def test_linemod_frames_match_reference(cuda_dev, mode):
    d = _linemod_batch(3)
    fib = _run_and_check(d, mode, 2024, cuda_dev)
    ok = fib.ok.cpu().numpy()
    assert list(ok) == [1, 1, 1, 0]
    ch = fib.choose[2, 0].cpu().numpy()
    assert np.array_equal(ch[3000:6000], ch[:3000])      # wrap duplicates


@pytest.mark.parametrize("mode", ["sampled", "full"])
def test_ycb_box_frames_with_holes_match_reference(cuda_dev, mode):
    _run_and_check(_ycb_batch(7), mode, 99, cuda_dev)


def test_seed_and_frame_index_change_the_subset(cuda_dev):
    d = _linemod_batch(5)
    d["depth"][1] = d["depth"][0]
    fib = FrameInputBuilder(4, N, normals="sampled", device=cuda_dev)
    args = [_t(d[k], cuda_dev) for k in ("depth", "K", "cam_scale", "rgb")]
    a = fib.build(*args, 1)[2].clone()
    b = fib.build(*args, 2)[2].clone()
    c = fib.build(*args, 1)[2]
    assert torch.equal(a, c) and not torch.equal(a[0], b[0]) and not torch.equal(a[0], a[1])


def test_build_under_cuda_graph_capture(cuda_dev):
    d = _ycb_batch(8)
    args = [_t(d[k], cuda_dev) for k in ("depth", "K", "cam_scale", "rgb")]
    eager = FrameInputBuilder(2, N, device=cuda_dev)
    want = [t.clone() for t in eager.build(*args, 5)]
    fib = FrameInputBuilder(2, N, device=cuda_dev)
    side = torch.cuda.Stream(cuda_dev)
    side.wait_stream(torch.cuda.current_stream(cuda_dev))
    with torch.cuda.stream(side):
        fib.build(*args, 5)                            # warm-up outside the capture
    torch.cuda.current_stream(cuda_dev).wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):                          # a host sync inside would fail the capture
        out = fib.build(*args, 5)
    for t in out:
        t.zero_()
    g.replay()
    torch.cuda.synchronize()
    for x, y in zip(out, want):
        assert torch.equal(x, y)


def test_estimate_normals_drop_in(cuda_dev):
    d = _ycb_batch(9)
    from oracle import depth_icp_oracle as dio

    cloud, valid = dio.dpt_2_cld(d["depth"][0], d["cam_scale"][0], d["K"][0])
    cld = cloud[valid][::20]
    got = estimate_normals(cld, device=cuda_dev)
    assert got.shape == (len(cld), 4) and got.dtype == np.float32
    idx = nr.knn(cld, cld)
    n, C, lam, curv = nr.normals(cld, idx, cld)
    sep = (lam[:, 1] - lam[:, 0]) / np.trace(C, axis1=1, axis2=2) >= 1e-3
    assert angle(got[sep, :3], n[sep]).max() <= 1e-6
    p = cld.astype(np.float64)
    clear = sep & (np.abs((n * p).sum(1)) >= 1e-6 * np.linalg.norm(p, axis=1))
    assert ((got[clear, :3].astype(np.float64) * n[clear]).sum(1) > 0).all()
    assert np.allclose(got[:, 3], curv, rtol=1e-5, atol=1e-7)
    assert not estimate_normals(cld[:49], device=cuda_dev).any()   # fewer than 50 points


def test_stand_in_network_runs_on_the_builders_output(cuda_dev):
    n = 4096
    d = _linemod_batch(11)
    fib = FrameInputBuilder(2, n, device=cuda_dev)
    cld, rgb, choose, pcld, ok = fib.build(*[_t(d[k][:2], cuda_dev) for k in ("depth", "K", "cam_scale", "rgb")], 3)
    model = testing.StandInPVN3D(n, seed=5).to(cuda_dev).eval()
    kp, seg, ctr = network.FusedPVN3D(model, cuda_dev).forward(cld, rgb / 255.0, choose)
    torch.cuda.synchronize()
    assert kp.shape == (2, model.num_kps, n, 3) and seg.shape[:2] == (2, n) and ctr.shape == (2, 1, n, 3)
    for t in (kp, seg, ctr):
        assert torch.isfinite(t).all()
    assert bool(ok.all())
