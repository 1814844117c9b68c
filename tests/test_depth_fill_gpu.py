"""DepthFiller (csrc/depth_fill.cu) against the numpy restatement of fill_missing (tests/depth_fill_ref.py) and the
goldens recorded from the reference: s4, s5, the pre-bilateral image and both top rows bit for bit, the bilateral
and the output within the bound of include/pvn3d_b200.h.  Every bit-exact comparison is paired with the wrong
references (depth_fill_ref.MUTANTS, and frame b answered with frame 0) it must reject.  Also: one batched call
equals single-frame calls, FrameInputBuilder(fill="multiscale") equals fill() then build(), CUDA graph capture,
and no host sync after warm-up."""
import os

import numpy as np
import pytest
import torch

import depth_fill_cases as dc
import depth_fill_ref as R
from pvn3d_b200 import synth
from pvn3d_b200.depth_fill import DepthFiller, fill_missing
from pvn3d_b200.frame_input import FrameInputBuilder

pytestmark = pytest.mark.gpu


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


@pytest.fixture(scope="module")
def cases(golden_dir):
    return dc.load(os.path.join(golden_dir, "fill_cases.npz"))


def _run(c, dev):
    depth = c["depth"]
    b, h, w = depth.shape
    f = DepthFiller(b, h, w, debug=True, device=dev)
    out = f.fill(_t(depth, dev), _t(c["cam_scale"], dev), float(c["scale_2_80m"]))
    torch.cuda.synchronize()
    return out.cpu().numpy(), f.stages.cpu().numpy(), f.top_rows.cpu().numpy()


@pytest.fixture(scope="module")
def results(cases, cuda_dev):
    """name -> (gpu out, gpu stages, gpu top rows, [oracle stages per frame])"""
    res = {}
    for name in dc.CASES:
        c = cases[name]
        s2s = np.float32(c["scale_2_80m"])
        ref = [R.fill_stages(c["depth"][b], c["cam_scale"][b], s2s) for b in range(c["depth"].shape[0])]
        res[name] = _run(c, cuda_dev) + (ref,)
    return res


@pytest.mark.parametrize("name", dc.CASES)
def test_stages_bit_exact(cases, results, name):
    c = cases[name]
    out, stages, tops, ref = results[name]
    for b, st in enumerate(ref):
        assert np.array_equal(stages[b, 0], st["s4"]) and np.array_equal(stages[b, 0], c["s4"][b]), (name, b, "s4")
        assert np.array_equal(stages[b, 1], st["s5"]) and np.array_equal(stages[b, 1], c["s5"][b]), (name, b, "s5")
        assert np.array_equal(stages[b, 2], st["s7_pre"]), (name, b, "pre-bilateral")
        assert np.array_equal(tops[b, 0], st["top1"]) and np.array_equal(tops[b, 1], st["top2"]), (name, b, "top")


@pytest.mark.parametrize("name", dc.CASES)
def test_bilateral_and_output_within_bound(cases, results, name):
    c = cases[name]
    out, stages, tops, ref = results[name]
    s2s = np.float32(c["scale_2_80m"])
    for b, st in enumerate(ref):
        bound = R.bilateral_bound(st["minmax"])
        e7 = np.abs(stages[b, 3].astype(np.float64) - st["s7"])
        assert e7.max() <= bound, (name, b, float(e7.max()), bound)
        # outside V the output is steps 1-9 and 11 only: bit-exact
        assert np.array_equal(out[b][~st["V"]], st["out"][~st["V"]]), (name, b)
        ro = st["out"].astype(np.float64)
        eo = np.abs(out[b] - ro)
        flips = int(((out[b] > 1e-6) != (st["out"] > 1e-6)).sum())
        print(f"{name}[{b}]: |bilateral - oracle| {e7.max():.2e} (bound {bound:.2e}), |out - oracle| {eo.max():.2e}, "
              f"validity flips {flips}")
        assert flips == 0, (name, b, flips)
        assert (eo <= R.out_bound(st["minmax"], c["cam_scale"][b], s2s, ro)).all(), (name, b, float(eo.max()))
        # against the reference's own output (at every OUT_STRIDE-th row and column for the YCB-shape frames)
        sub = slice(None) if "out" in c else slice(None, None, dc.OUT_STRIDE)
        rec = c["out"][b] if "out" in c else c["out_sub"][b]
        er = np.abs(out[b][sub, sub] - rec.astype(np.float64))
        assert (er <= R.out_bound(st["minmax"], c["cam_scale"][b], s2s, ro[sub, sub])).all(), (name, b, float(er.max()))


def test_wrong_references_are_rejected(cases, results):
    """each mutant differs from the kernel's output on some case: a bit-exact stage (s4, s5, the pre-bilateral
    image) differs, or the bilateral is farther than the bound; and frame b is not frame 0's answer"""
    told = {m: [] for m in R.MUTANTS}
    for name in dc.CASES:
        c = cases[name]
        out, stages, tops, ref = results[name]
        s2s = np.float32(c["scale_2_80m"])
        for b, st in enumerate(ref):
            for m in R.MUTANTS:
                mst = R.fill_stages(c["depth"][b], c["cam_scale"][b], s2s, mutant=m)
                if not np.array_equal(stages[b, 2], mst["s7_pre"]) or \
                        R.mutant_rejected(mst, stages[b, 0], stages[b, 1], stages[b, 3], st["minmax"]):
                    told[m].append(f"{name}[{b}]")
            if b > 0:   # frame b answered with frame 0
                assert not np.array_equal(stages[b, 2], ref[0]["s7_pre"]) or name == "all_zero", (name, b)
    print({m: v for m, v in told.items()})
    for m, v in told.items():
        assert v, m


def _batch16():
    z = dc.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fill_cases.npz"))["ycb"]
    rng = np.random.default_rng(3)
    depth = np.stack([z["depth"][i % len(z["depth"])] for i in range(16)]).astype(np.float32)
    for i in range(16):
        y, x = rng.integers(0, 400), rng.integers(0, 560)
        depth[i, y:y + int(rng.integers(10, 80)), x:x + int(rng.integers(10, 80))] = 0
        depth[i][rng.random((480, 640)) < 0.02 * (i % 4)] = 0
    cs = np.array([10000, 10000, 3800, 8000] * 4, np.float32)
    return depth, cs


def test_batch_equals_single_frames(cuda_dev):
    depth, cs = _batch16()
    fb = DepthFiller(16, debug=True, device=cuda_dev)
    out = fb.fill(_t(depth, cuda_dev), _t(cs, cuda_dev)).clone()
    st, tops = fb.stages.clone(), fb.top_rows.clone()
    f1 = DepthFiller(1, debug=True, device=cuda_dev)
    for i in range(16):
        o1 = f1.fill(_t(depth[i:i + 1], cuda_dev), _t(cs[i:i + 1], cuda_dev))
        assert torch.equal(o1[0], out[i]) and torch.equal(f1.stages[0], st[i]) and torch.equal(f1.top_rows[0], tops[i])
    # frame b is its own answer, not frame 0's
    assert not torch.equal(out[1], out[0]) and not torch.equal(out[5], out[0])
    # the one-frame numpy drop-in is the same computation
    assert np.array_equal(fill_missing(depth[2], cs[2], 1), out[2].cpu().numpy())


def test_frame_input_builder_fill_equals_fill_then_build(cuda_dev):
    depth, cs = _batch16()
    depth, cs = depth[:4], cs[:4]
    rng = np.random.default_rng(5)
    K = np.repeat(synth.K_YCB1.astype(np.float32)[None], 4, 0)
    rgb = rng.integers(0, 256, (4, 3, 480, 640), dtype=np.uint8)
    args = (_t(K, cuda_dev), _t(cs, cuda_dev), _t(rgb, cuda_dev))
    fib = FrameInputBuilder(4, 12288, fill="multiscale", device=cuda_dev)
    got = [t.clone() for t in fib.build(_t(depth, cuda_dev), args[0], args[1], args[2], 9)]
    filled = DepthFiller(4, device=cuda_dev).fill(_t(depth, cuda_dev), args[1]).clone()
    assert torch.equal(fib.filled[:4], filled)
    want = FrameInputBuilder(4, 12288, device=cuda_dev).build(filled, args[0], args[1], args[2], 9)
    for x, y in zip(got, want):
        assert torch.equal(x, y)
    # filling changes the input: more valid pixels, so a different subset
    plain = FrameInputBuilder(4, 12288, device=cuda_dev).build(_t(depth, cuda_dev), args[0], args[1], args[2], 9)
    assert not torch.equal(plain[2], got[2])
    with pytest.raises(ValueError):
        FrameInputBuilder(1, 12288, fill="fast", device=cuda_dev)


def test_fill_under_graph_capture_and_without_host_sync(cuda_dev):
    depth, cs = _batch16()
    d, c = _t(depth[:4], cuda_dev), _t(cs[:4], cuda_dev)
    want = DepthFiller(4, device=cuda_dev).fill(d, c).clone()
    f = DepthFiller(4, device=cuda_dev)
    side = torch.cuda.Stream(cuda_dev)
    side.wait_stream(torch.cuda.current_stream(cuda_dev))
    with torch.cuda.stream(side):
        f.fill(d, c)                                    # warm-up outside the capture
    torch.cuda.current_stream(cuda_dev).wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):                           # a host sync inside would fail the capture
        out = f.fill(d, c)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    torch.cuda.set_sync_debug_mode("error")
    try:
        again = f.fill(d, c)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert torch.equal(again, want)
