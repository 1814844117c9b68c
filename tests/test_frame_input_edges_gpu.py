"""csrc/normals.cu at its edges on the GPU.  pvn3d_frame_sample and pvn3d_knn_normals are called through _lib on the
current stream, with workspaces from their size queries, on the cases of tests/frame_input_cases.py:
  * the sampler's choose, ok, columns 0..5, pcld and labels bit for bit against tests/normals_ref.py, columns 6 and
    up untouched, and every sampler mutant rejected on the kernel's output;
  * the 50 neighbour indices index for index against plain brute force (-1 rows included), the normals under the
    contract of frame_input_cases.normal_faults, and every kNN and normal mutant rejected on the kernel's output;
  * the call's optional outputs, row strides, repeatability and mixed frame_ok;
  * FrameInputBuilder with fewer frames than it was made for, and in "full" mode on frames where all 307200 pixels
    are valid (one with a spurious 65 m pixel), every query checked against a float64 brute force on the GPU;
  * estimate_normals on NaN rows and on clouds of 49, 50 and 51 points.
Takes about 21 s on an H100 (45 tests), most of it in the host references and the GPU brute force."""
import numpy as np
import pytest
import torch

import frame_input_cases as fc
import normals_ref as nr
from pvn3d_b200 import _lib, synth
from pvn3d_b200._lib import check, ptr
from pvn3d_b200.frame_input import FrameInputBuilder, estimate_normals

pytestmark = pytest.mark.gpu

N = 12288
U32 = np.uint32
SENTINEL = U32(0x7FC0DEAD)          # a NaN with a payload, in every output column a call must not write


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _sentinel(shape, dev):
    return _t(np.full(shape, SENTINEL, U32).view(np.float32), dev)


def _ws(nbytes, dev):
    """(owner, 256-B aligned address) of a workspace of nbytes"""
    assert nbytes > 0
    buf = torch.empty(int(nbytes) + 256, dtype=torch.uint8, device=dev)
    return buf, (buf.data_ptr() + 255) // 256 * 256


@pytest.fixture(scope="module")
def lib(cuda_dev):
    return _lib.load()


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


# ---- pvn3d_frame_sample ---------------------------------------------------------------------------------------
def run_sample(lib, dev, case, data):
    cloud, rgb, lab = data
    valid, n, stride = case["valid"], case["n"], case["stride"]
    b, hw = valid.shape
    cld = _sentinel((b, n, stride), dev)
    pcld = torch.full((b, n, 3), float("nan"), device=dev)
    choose = torch.full((b, n), -7, dtype=torch.int64, device=dev)
    ok = torch.full((b,), 7, dtype=torch.uint8, device=dev)
    labels = torch.full((b, n), -7, dtype=torch.int32, device=dev) if lab is not None else None
    c_t, v_t, r_t = _t(cloud, dev), _t(valid.astype(np.uint8), dev), _t(rgb, dev)
    l_t = _t(lab, dev) if lab is not None else None
    nbytes = lib.pvn3d_frame_sample_workspace_bytes(b, hw, n)
    buf, addr = _ws(nbytes, dev)
    check(lib.pvn3d_frame_sample(ptr(c_t), ptr(v_t), ptr(r_t), case["rgb_u8"], ptr(l_t), b, hw, n, case["seed"],
                                 ptr(cld), stride, ptr(pcld), ptr(choose), ptr(labels), ptr(ok), addr, nbytes,
                                 _stream(dev)), "pvn3d_frame_sample")
    torch.cuda.synchronize(dev)
    return dict(cld=cld.cpu().numpy(), pcld=pcld.cpu().numpy(), choose=choose.cpu().numpy(), ok=ok.cpu().numpy(),
                labels=None if labels is None else labels.cpu().numpy())


@pytest.fixture(scope="module")
def sampled(lib, cuda_dev):
    """name -> (case, reference, kernel output) for every sampler case"""
    res = {}
    for name in fc.SAMPLE_CASES:
        case = fc.sample_case(name)
        data = fc.sample_data(case)
        res[name] = (case, fc.sample_ref(case, data), run_sample(lib, cuda_dev, case, data))
    return res


@pytest.mark.parametrize("name", list(fc.SAMPLE_CASES))
def test_sampler_matches_reference(sampled, name):
    case, want, got = sampled[name]
    assert np.array_equal(got["ok"], want["ok"])
    assert np.array_equal(got["choose"], want["choose"])
    cld = got["cld"].view(U32)
    assert np.array_equal(cld[:, :, :6], want["cld6"].view(U32))
    assert (cld[:, :, 6:] == SENTINEL).all()                       # columns 6 and up are the normals' call's
    assert np.array_equal(got["pcld"].view(U32), want["cld6"][:, :, :3].view(U32))
    if got["labels"] is not None:
        assert np.array_equal(got["labels"], want["labels"])
    off = got["ok"] == 0
    assert not got["choose"][off].any() and not cld[off, :, :6].any() and not got["pcld"].view(U32)[off].any()
    if got["labels"] is not None:
        assert not got["labels"][off].any()


@pytest.mark.parametrize("mutant", fc.SAMPLE_MUTANTS)
def test_sampler_mutants_are_rejected(sampled, mutant):
    assert any(fc.sample_mutant_differs(mutant, case, got["choose"], got["ok"])
               for case, _, got in sampled.values()), mutant


# ---- pvn3d_knn_normals ----------------------------------------------------------------------------------------
def run_knn(lib, dev, ref, valid, query, *, frame_ok=None, stride=3, curv=True, n64=True, nn=True):
    b, r, _ = ref.shape
    q = query.shape[1]
    ref_t, q_t = _t(ref, dev), _t(query, dev)
    v_t = None if valid is None else _t(np.asarray(valid, np.uint8), dev)
    ok_t = None if frame_ok is None else _t(np.asarray(frame_ok, np.uint8), dev)
    out = _sentinel((b, q, stride), dev)
    curv_t = torch.full((b, q), float("nan"), device=dev) if curv else None
    n64_t = torch.full((b, q, 3), float("nan"), dtype=torch.float64, device=dev) if n64 else None
    nn_t = torch.full((b, q, fc.K), -7, dtype=torch.int32, device=dev) if nn else None
    nbytes = lib.pvn3d_knn_normals_workspace_bytes(b, r, q)
    buf, addr = _ws(nbytes, dev)
    check(lib.pvn3d_knn_normals(ptr(ref_t), ptr(v_t), r, ptr(q_t), q, b, ptr(ok_t), ptr(out), stride, ptr(curv_t),
                                ptr(n64_t), ptr(nn_t), addr, nbytes, _stream(dev)), "pvn3d_knn_normals")
    torch.cuda.synchronize(dev)
    get = lambda t: None if t is None else t.cpu().numpy()   # noqa: E731
    return dict(out=get(out), curv=get(curv_t), n64=get(n64_t), nn=get(nn_t))


def brute_knn(ref, valid, query, chunk=256):
    """[B,Q,50] int64 on ref's device: float64 brute force, one torch op per step (nothing contracts).  The 50th
    smallest d2 is found first; every candidate at or below it is then ranked by (d2, index) without relying on
    topk's order among ties.  -1 rows for a non-finite query or fewer than 50 usable points."""
    b, _, _ = ref.shape
    q = query.shape[1]
    out = torch.full((b, q, fc.K), -1, dtype=torch.int64, device=ref.device)
    inf = torch.tensor(float("inf"), dtype=torch.float64, device=ref.device)
    for f in range(b):
        p = ref[f].double()
        use = torch.isfinite(p).all(1)
        if valid is not None:
            use &= valid[f].bool()
        if int(use.sum()) < fc.K:
            continue
        for s in range(0, q, chunk):
            qq = query[f, s:s + chunk].double()
            fin = torch.isfinite(qq).all(1)
            qq = torch.where(fin[:, None], qq, torch.zeros_like(qq))
            dx = torch.sub(qq[:, None, 0], p[None, :, 0])
            dy = torch.sub(qq[:, None, 1], p[None, :, 1])
            dz = torch.sub(qq[:, None, 2], p[None, :, 2])
            d2 = torch.add(torch.add(torch.mul(dx, dx), torch.mul(dy, dy)), torch.mul(dz, dz))
            d2 = torch.where(use[None], d2, inf)
            kth = torch.topk(d2, fc.K, dim=1, largest=False).values[:, -1:]
            cand = d2 <= kth
            m = int(cand.sum(1).max())
            v, i = torch.topk(torch.where(cand, d2, inf), m, dim=1, largest=False)
            i, o = torch.sort(i, dim=1)                              # index order, then a stable sort by d2
            v = torch.gather(v, 1, o)
            v, o = torch.sort(v, dim=1, stable=True)
            i = torch.gather(i, 1, o)[:, :fc.K]
            out[f, s:s + chunk] = torch.where(fin[:, None], i, torch.full_like(i, -1))
    return out


def _check_normals(n32, n64, curv, C, lam, want, want_curv, q, stats):
    """the float32 normal is the rounded float64 one, and the float64 one keeps the contract"""
    assert np.array_equal(n32.reshape(-1, 3).view(U32), n64.reshape(-1, 3).astype(np.float32).view(U32))
    faults, worst = fc.normal_faults(n64.reshape(-1, 3), curv.reshape(-1), C, lam, want, want_curv, q.reshape(-1, 3))
    for k, v in worst.items():
        stats[k] = max(stats.get(k, 0.0), v)
    assert faults == [], (faults, worst)


@pytest.mark.parametrize("name", list(fc.KNN_CASES))
def test_knn_case(lib, cuda_dev, name):
    build, knn_mutants, normal_mutants = fc.KNN_CASES[name]
    inputs = build()
    gots, stats = [], {}
    for inp in inputs:
        ref, valid, q = inp
        got = run_knn(lib, cuda_dev, *inp)
        want = np.stack([nr.knn_brute(ref[f], q[f], None if valid is None else valid[f]) for f in range(len(ref))])
        assert np.array_equal(got["nn"], want)
        n, C, lam, curv = fc.normals_of(inp, want)
        _check_normals(got["out"], got["n64"], got["curv"], C, lam, n, curv, q, stats)
        gots.append(got)
    print(f"\n{name}: " + ", ".join(f"worst {k} {v:.3e}" for k, v in stats.items()))
    for m in knn_mutants:
        assert any(not np.array_equal(fc.knn_mutant(m, inp), g["nn"]) for inp, g in zip(inputs, gots)), m
    for m in normal_mutants:
        assert any(fc.normal_mutant_faults(m, inp, g["nn"].astype(np.int64)) for inp, g in zip(inputs, gots)), m
    if name == "extremes":
        n64 = gots[0]["n64"]
        assert (n64[2] == [0.0, 0.0, 1.0]).all()        # the wall through the origin: n . q = 0, not flipped
        assert (n64[3][:, 0] == 0).all()                # the line along x: lambda0 = lambda1 = 0, n orthogonal to it
        assert not gots[0]["curv"][3].any()
    if name == "coincident_wrap":
        on = (inputs[0][2][0] == inputs[0][0][0, 100]).all(1)
        assert on.sum() == 60 and not gots[0]["n64"][0][on].any()   # trace 0: exact zeros


def test_knn_optional_outputs_and_strides(lib, cuda_dev):
    inp = fc.KNN_CASES["ties"][0]()[0]
    full = run_knn(lib, cuda_dev, *inp)
    for kw in (dict(curv=False, n64=False, nn=False), dict(curv=True, n64=False, nn=False),
               dict(curv=False, n64=True, nn=False), dict(curv=False, n64=False, nn=True)):
        assert np.array_equal(run_knn(lib, cuda_dev, *inp, **kw)["out"].view(U32), full["out"].view(U32)), kw
    for stride in (4, 9, 16):
        got = run_knn(lib, cuda_dev, *inp, stride=stride)["out"].view(U32)
        assert np.array_equal(got[:, :, :3], full["out"].view(U32))
        assert (got[:, :, 3:] == SENTINEL).all()


def test_knn_calls_are_repeatable(lib, cuda_dev):
    # 30-31 copies of every point: the scatter's atomics order each cell differently from call to call
    for inp in fc.KNN_CASES["coincident_wrap"][0]() + fc.KNN_CASES["scales"][0]():
        a, b = run_knn(lib, cuda_dev, *inp), run_knn(lib, cuda_dev, *inp)
        for k in a:
            assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k


def test_knn_mixed_frame_ok(lib, cuda_dev):
    inp = fc.KNN_CASES["usable_counts"][0]()[0]
    all_ok = run_knn(lib, cuda_dev, *inp)
    fok = np.array([1, 0, 1, 0, 1], np.uint8)
    got = run_knn(lib, cuda_dev, *inp, frame_ok=fok)
    on, off = fok == 1, fok == 0
    for k in ("out", "curv", "n64", "nn"):
        assert np.array_equal(got[k][on].view(np.uint8), all_ok[k][on].view(np.uint8)), k
    assert (got["nn"][off] == -1).all()
    assert not got["out"][off].any() and not got["curv"][off].any() and not got["n64"][off].any()


# ---- FrameInputBuilder ------------------------------------------------------------------------------------------
def _all_valid_depth(b, seed):
    """LineMOD-shape frames in mm where every pixel is valid: spheres over a plane"""
    rng = np.random.default_rng(seed)
    K = synth.K_LINEMOD.astype(np.float64)
    depth = np.stack([np.round(synth._render(K, [np.array([0.05, -0.02, 0.8]), np.array([-0.1, 0.05, 0.9])],
                                             [0.06, 0.09], rng)[0] * 1000.0) for _ in range(b)]).astype(np.float32)
    assert (depth > 0).all()
    rgb = rng.integers(0, 256, size=(b, 3, synth.H, synth.W), dtype=np.uint8)
    return dict(depth=depth, K=np.repeat(K.astype(np.float32)[None], b, 0), cam_scale=np.full(b, 1000.0, np.float32),
                rgb=rgb)


def _build(fib, d, seed, dev):
    return fib.build(*[_t(d[k], dev) for k in ("depth", "K", "cam_scale", "rgb")], seed)


def _check_full_build(fib, d, seed, stats):
    """every query of a "full" build against the GPU brute force, and its normals against the contract"""
    b = len(d["depth"])
    ok = fib.ok[:b].cpu().numpy()
    assert ok.all()
    valid = fib.valid[:b].cpu().numpy().astype(bool)
    assert valid.all()
    ch = fib.choose[:b, 0].cpu().numpy()
    for f in range(b):
        assert np.array_equal(ch[f], nr.sample_frame(valid[f], N, seed, f)[0])
    want = brute_knn(fib.cloud[:b], fib.valid[:b], fib.pcld[:b]).cpu().numpy()
    assert np.array_equal(fib.nn_idx[:b].cpu().numpy(), want)
    cloud, pcld = fib.cloud[:b].cpu().numpy(), fib.pcld[:b].cpu().numpy()
    n, C, lam, curv = fc.normals_of((cloud, None, pcld), want)
    _check_normals(fib.cld_rgb_nrm[:b, :, 6:].cpu().numpy(), fib.normals64[:b].cpu().numpy(),
                   fib.curvature[:b].cpu().numpy(), C, lam, n, curv, pcld, stats)


def test_build_with_fewer_frames_than_made_for(cuda_dev):
    d = _all_valid_depth(2, 20)
    d["depth"][1, ::2] = 0.0                                     # half the rows invalid
    small = FrameInputBuilder(2, N, normals="sampled", debug=True, device=cuda_dev)
    want = [t.clone() for t in _build(small, d, 4, cuda_dev)]
    big = FrameInputBuilder(5, N, normals="sampled", debug=True, device=cuda_dev)
    got = _build(big, d, 4, cuda_dev)
    for x, y in zip(got, want):
        assert x.shape == y.shape and torch.equal(x.view(torch.uint8), y.view(torch.uint8))
    for a in ("nn_idx", "normals64", "curvature"):
        assert torch.equal(getattr(big, a)[:2], getattr(small, a))
    assert torch.equal(big.nn_idx[:2].long(), brute_knn(big.pcld[:2], None, big.pcld[:2]))


def test_full_mode_on_all_valid_frames(cuda_dev):
    d = _all_valid_depth(2, 21)
    fib = FrameInputBuilder(2, N, normals="full", debug=True, device=cuda_dev)
    _build(fib, d, 6, cuda_dev)
    stats = {}
    _check_full_build(fib, d, 6, stats)
    print("\nfull, 307200 valid: " + ", ".join(f"worst {k} {v:.3e}" for k, v in stats.items()))


def test_full_mode_with_a_65m_pixel(cuda_dev):
    d = _all_valid_depth(2, 22)
    d["depth"][0, 240, 320] = 65000.0                            # one spurious pixel 65 m away: a coarse grid
    fib = FrameInputBuilder(2, N, normals="full", debug=True, device=cuda_dev)
    _build(fib, d, 8, cuda_dev)                                  # warm-up
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    _build(fib, d, 8, cuda_dev)
    t1.record()
    torch.cuda.synchronize()
    stats = {}
    _check_full_build(fib, d, 8, stats)
    print(f"\nfull with a 65 m pixel: build() {t0.elapsed_time(t1):.2f} ms for 2 frames (not asserted); "
          + ", ".join(f"worst {k} {v:.3e}" for k, v in stats.items()))


# ---- estimate_normals -------------------------------------------------------------------------------------------
def test_estimate_normals_nan_rows_and_small_clouds(cuda_dev):
    rng = np.random.default_rng(23)
    cld = rng.normal(size=(500, 3)).astype(np.float32)
    cld[::37, 1] = np.nan
    cld[5] = np.inf
    bad = ~np.isfinite(cld).all(1)
    got = estimate_normals(cld, device=cuda_dev)
    assert not got[bad].any()
    stats = {}
    for m in (49, 50, 51, 500):
        c = cld if m == 500 else rng.normal(size=(m, 3)).astype(np.float32) + np.float32(0.5)
        g = got if m == 500 else estimate_normals(c, device=cuda_dev)
        assert g.shape == (m, 4) and g.dtype == np.float32
        idx = nr.knn_brute(c, c)
        if m == 49:
            assert (idx == -1).all() and not g.any()
            continue
        n, C, lam, curv = nr.normals(c, idx, c)
        faults, worst = fc.normal_faults(g[:, :3], g[:, 3], C, lam, n, curv, c)
        # the float32 normal is within 2^-24 of unit length, not 1e-12, and so is its residual: the rest holds as is
        assert set(faults) <= {"unit", "residual"}, (m, faults, worst)
        fin = np.isfinite(c).all(1)
        assert np.abs(np.linalg.norm(g[fin, :3].astype(np.float64), axis=1) - 1).max() <= 3 * 2.0 ** -24
        stats[m] = {k: f"{v:.3e}" for k, v in worst.items()}
    print(f"\nestimate_normals: {stats}")
