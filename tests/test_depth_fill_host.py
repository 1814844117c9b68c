"""The numpy restatement of fill_missing (tests/depth_fill_ref.py) against the goldens recorded from the reference,
and against cv2 where it is installed; the C ABI's refusals of csrc/depth_fill.cu before any launch; the
options fill_missing accepts.  No GPU needed."""
import ctypes
import os

import numpy as np
import pytest

import depth_fill_cases as dc
import depth_fill_ref as R
from pvn3d_b200 import _lib
from pvn3d_b200.depth_fill import fill_missing


@pytest.fixture(scope="module")
def cases(golden_dir):
    return dc.load(os.path.join(golden_dir, "fill_cases.npz"))


def test_goldens_hold_every_case(cases):
    assert sorted(cases) == sorted(dc.CASES)


@pytest.mark.parametrize("name", dc.CASES)
def test_oracle_matches_reference_goldens(cases, name):
    c = cases[name]
    s2s = np.float32(c["scale_2_80m"])
    for b in range(c["depth"].shape[0]):
        st = R.fill_stages(c["depth"][b], c["cam_scale"][b], s2s)
        for k in ("s1", "s2", "s3", "s4", "s5"):
            if k in c:
                assert np.array_equal(st[k], c[k][b]), (name, b, k)
        if "s7" in c:
            assert np.abs(st["s7"].astype(np.float64) - c["s7"][b]).max() <= R.bilateral_bound(st["minmax"])
        got, ref = (st["out"], c["out"][b]) if "out" in c else \
            (st["out"][::dc.OUT_STRIDE, ::dc.OUT_STRIDE], c["out_sub"][b])
        ref = ref.astype(np.float64)
        assert (np.abs(got - ref) <= R.out_bound(st["minmax"], c["cam_scale"][b], s2s, ref)).all()


def test_every_mutant_is_told_apart_by_some_golden(cases):
    for m in R.MUTANTS:
        told = False
        for name in dc.CASES:
            c = cases[name]
            if "s7" not in c:
                continue
            for b in range(c["depth"].shape[0]):
                st = R.fill_stages(c["depth"][b], c["cam_scale"][b], np.float32(c["scale_2_80m"]))
                mst = R.fill_stages(c["depth"][b], c["cam_scale"][b], np.float32(c["scale_2_80m"]), mutant=m)
                told |= R.mutant_rejected(mst, c["s4"][b], c["s5"][b], c["s7"][b], st["minmax"])
        if m == "dilate_zero":   # only a large region beyond 3 m shows it: the YCB frame read with cam_scale 3800
            c = cases["ycb"]
            mst = R.fill_stages(c["depth"][1], c["cam_scale"][1], mutant=m)
            told |= not (np.array_equal(mst["s4"], c["s4"][1]) and np.array_equal(mst["s5"], c["s5"][1]))
        assert told, m


# ---- the restatement's primitives against cv2 ---------------------------------------------------------------------
def _frames(seed, n=3):
    rng = np.random.default_rng(seed)
    for _ in range(n):
        h, w = int(rng.integers(5, 60)), int(rng.integers(5, 60))
        a = rng.uniform(-2, 3, (h, w)).astype(np.float32)
        a[rng.random((h, w)) < 0.3] = 0
        yield a


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_primitives_match_cv2(seed):
    cv2 = pytest.importorskip("cv2")
    for a in _frames(seed):
        for k, mask in ((3, R.CROSS_3), (5, R.CROSS_5), (7, R.CROSS_7), (5, R.FULL_5), (9, R.FULL_9)):
            kern = mask.astype(np.uint8)
            assert np.array_equal(R.dilate(a, mask), cv2.dilate(a, kern)), k
            assert np.array_equal(R.erode(a, mask), cv2.erode(a, kern)), k
        assert np.array_equal(R.erode(R.dilate(a, R.FULL_5), R.FULL_5),
                              cv2.morphologyEx(a, cv2.MORPH_CLOSE, R.FULL_5.astype(np.uint8)))
        assert np.array_equal(R.median5(a), cv2.medianBlur(a, 5))
        got, mm = R.bilateral(a)
        assert np.abs(got.astype(np.float64) - cv2.bilateralFilter(a, 5, 0.5, 2.0)).max() <= R.bilateral_bound(mm)


def test_bilateral_copy_path_and_taps():
    cv2 = pytest.importorskip("cv2")
    a = np.full((12, 16), 1.25, np.float32)
    got, mm = R.bilateral(a)
    assert np.array_equal(got, a)
    # cv2 builds may filter a constant image instead of copying it; either way it stays within the bound
    assert np.abs(cv2.bilateralFilter(a, 5, 0.5, 2.0).astype(np.float64) - a).max() <= R.bilateral_bound(mm)
    taps = R.space_taps()
    assert len(taps) == 13 and all(dy * dy + dx * dx <= 4 for dy, dx, _ in taps)


# ---- the ABI refuses what it cannot do before launching anything ------------------------------------------------
def _fake(i=1):
    return ctypes.c_void_p(256 * i)           # never dereferenced: every call below returns before a launch


def test_workspace_query_refuses_bad_sizes():
    lib = _lib.load()
    assert lib.pvn3d_depth_fill_workspace_bytes(16, 480, 640) >= 2 * 16 * 480 * 640 * 4
    assert lib.pvn3d_depth_fill_workspace_bytes(7000, 480, 640) == 0        # B*H*W >= 2^31
    assert lib.pvn3d_depth_fill_workspace_bytes(0, 480, 640) == 0
    assert lib.pvn3d_depth_fill_workspace_bytes(1, 0, 640) == 0
    assert lib.pvn3d_depth_fill_workspace_bytes(1, 480, -1) == 0
    assert lib.pvn3d_depth_fill_workspace_bytes(70000, 4, 4) == 0           # B > 65535


def test_entry_point_refuses_before_launch():
    lib = _lib.load()
    big = 1 << 40
    f = _fake
    ok = lib.pvn3d_depth_fill_workspace_bytes(2, 480, 640)
    assert lib.pvn3d_depth_fill(f(1), f(2), 1.0, 7000, 480, 640, f(3), None, None, f(4), big, None) == -2
    assert lib.pvn3d_depth_fill(f(1), f(2), 1.0, 70000, 4, 4, f(3), None, None, f(4), big, None) == -2
    assert lib.pvn3d_depth_fill(None, f(2), 1.0, 2, 480, 640, f(3), None, None, f(4), big, None) == -1
    assert lib.pvn3d_depth_fill(f(1), None, 1.0, 2, 480, 640, f(3), None, None, f(4), big, None) == -1
    assert lib.pvn3d_depth_fill(f(1), f(2), 1.0, 2, 480, 640, None, None, None, f(4), big, None) == -1
    assert lib.pvn3d_depth_fill(f(1), f(2), 1.0, 2, 480, 640, f(3), None, None, None, big, None) == -1
    assert lib.pvn3d_depth_fill(f(1), f(2), 1.0, 0, 480, 640, f(3), None, None, f(4), big, None) == -1
    assert lib.pvn3d_depth_fill(f(1), f(2), 0.0, 2, 480, 640, f(3), None, None, f(4), big, None) == -1
    assert lib.pvn3d_depth_fill(f(1), f(2), float("nan"), 2, 480, 640, f(3), None, None, f(4), big, None) == -1
    assert lib.pvn3d_depth_fill(f(1), f(2), 1.0, 2, 480, 640, f(3), None, None, f(4), ok - 1, None) == -4
    assert lib.pvn3d_depth_fill(f(1), f(2), 1.0, 2, 480, 640, f(3), None, None, ctypes.c_void_p(257), big,
                                None) == -1                                  # workspace not 256-B aligned


@pytest.mark.parametrize("kw", [dict(fill_type="fast"), dict(fill_type="bogus"), dict(extrapolate=True),
                                dict(blur_type="gaussian"), dict(blur_type="none")])
def test_fill_missing_refuses_other_options(kw):
    with pytest.raises(ValueError):
        fill_missing(np.zeros((8, 8), np.float32), 10000.0, 1, **kw)
