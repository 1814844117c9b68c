"""Inputs of the depth-fill goldens (tests/golden/make_golden_fill.py) and tests: small frames at the edges of
fill_in_multiscale's rules, and YCB-shape 480x640 frames from synth.make_icp_depth_batch with dropout and holes.
Every case is (name, depth [B,H,W] f32 raw units, cam_scale [B] f32, scale_2_80m, stages to record).

The YCB-shape frames are stored losslessly but compactly (encode_large / load): depth as row differences,
s5 as the pixels where it differs from s4, and the output at every OUT_STRIDE-th row and column only
("out_sub"); load() restores depth, s4 and s5 bit for bit."""
from __future__ import annotations

import numpy as np

CS = np.float32(10000.0)
SMALL = ("s3", "s4", "s5", "s7", "out")
LARGE = ("s4", "s5", "out_sub")
OUT_STRIDE = 8
CASES = ("all_zero", "single_pixel", "empty_columns", "thresholds", "loop_at_t", "borders", "constant",
         "top_spike", "far_border", "scales", "ycb")


def _block(h, w, value, rows, cols):
    d = np.zeros((h, w), np.float32)
    d[rows[0]:rows[1], cols[0]:cols[1]] = value
    return d


def _u(rng, lo, hi, shape):
    """integer raw depths, as a depth PNG holds them"""
    return np.round(rng.uniform(lo, hi, shape)).astype(np.float32)


def make_cases():
    rng = np.random.default_rng(7)
    out = []
    # nothing valid: every stage is zero and the bilateral takes the copy path
    out.append(("all_zero", np.zeros((1, 24, 32), np.float32), np.array([CS]), 1.0, SMALL))
    one = np.zeros((1, 24, 32), np.float32)
    one[0, 13, 17] = 12000
    out.append(("single_pixel", one, np.array([CS]), 1.0, SMALL))
    # columns with no valid pixel, empty top rows, a ragged top edge
    d = _u(rng, 6000, 16000, (40, 48))
    d[rng.random(d.shape) < 0.3] = 0
    d[:9] = 0
    for c in range(48):
        d[: int(rng.integers(9, 20)), c] = 0
    d[:, 5:7] = 0
    d[:, 30] = 0
    d[:, 44:] = 0
    out.append(("empty_columns", d[None], np.array([CS]), 1.0, SMALL))
    # d exactly 0.01, 1, 2, 3 after the division, and beyond 3 m
    vals = np.array([0, 100, 100, 10000, 20000, 30000, 35000, 60000, 9999, 10001, 19999, 20001, 29999, 5000, 15000,
                     25000], np.float32)
    d = vals[rng.integers(0, len(vals), (40, 48))]
    d[rng.random(d.shape) < 0.4] = 0
    out.append(("thresholds", d[None], np.array([CS]), 1.0, SMALL))
    # a pixel equal to 0.01f (raw 100 / 10000) in the middle of a hole the six iterations reach
    d = np.full((48, 48), 14000, np.float32)
    d[8:40, 8:40] = 0
    d[24, 24] = 100
    d2 = d.copy()
    d2[20:28, 20:28] = 0
    d2[24, 24] = 100
    d2[22, 27] = 100
    out.append(("loop_at_t", np.stack([d, d2]), np.array([CS, CS]), 1.0, SMALL))
    # holes on every border and holes too large for six iterations
    d = _u(rng, 5000, 25000, (64, 80))
    d[rng.random(d.shape) < 0.2] = 0
    d[0:3, 10:30] = 0
    d[-4:, 40:70] = 0
    d[20:40, 0:5] = 0
    d[5:25, -6:] = 0
    d[0:6, 0:6] = 0
    d[-6:, -6:] = 0
    d[25:60, 25:60] = 0
    out.append(("borders", d[None], np.array([CS]), 1.0, SMALL))
    # constant everywhere: the bilateral's copy path
    out.append(("constant", np.full((1, 24, 32), 15000, np.float32), np.array([CS]), 1.0, SMALL))
    # valid pixels that sit just under their column's top with empty columns around them: the median turns
    # them invalid, so V before and after the median differ; a constant valid block under an empty top, whose
    # valid-only min / max would be equal
    d = np.zeros((32, 40), np.float32)
    d[20:, :] = 25000
    d[12, 8] = d[12, 20] = 14000
    d[14:20, 30] = 14000
    d2 = _block(32, 40, 25000, (16, 32), (0, 40))
    out.append(("top_spike", np.stack([d, d2]), np.array([CS, CS]), 1.0, SMALL))
    # depth beyond 3 m against the borders: negative values there, which the dilations must not raise to 0
    d = _u(rng, 31000, 60000, (32, 40))
    d[rng.random(d.shape) < 0.3] = 0
    d[10:22, 12:28] = _u(rng, 8000, 28000, (12, 16))
    d[0, :] = 0
    d[:, 0] = 0
    out.append(("far_border", d[None], np.array([CS]), 1.0, SMALL))
    # a different cam_scale per frame and scale_2_80m != 1
    d = _u(rng, 3000, 9000, (3, 40, 48))
    d[rng.random(d.shape) < 0.35] = 0
    d[:, 10:22, 12:30] = 0
    out.append(("scales", d, np.array([4000, 5000, 2500], np.float32), 1.7, SMALL))
    out.append(("ycb",) + _ycb_frames() + (1.0, LARGE))
    return out


def _ycb_frames():
    from pvn3d_b200 import synth

    # without depth noise, so that the recorded stages compress; dropout and hole boxes as usual
    batch = synth.make_icp_depth_batch(2, n_obj=3, seed=11, hole_frac=0.05, n_hole_boxes=4, noise=0.0)
    depth = batch["depth"].astype(np.float32)
    # the second frame read with a smaller cam_scale (deeper, some of it beyond 3 m)
    cs = np.array([10000, 3800], np.float32)
    return depth, cs


def encode_large(name, arrays):
    """{key: array} of one YCB-shape case -> the npz entries that load() restores"""
    out = {}
    d = arrays["depth"]
    assert np.array_equal(d, np.round(d)) and 0 <= d.min() and d.max() < 2**31
    step = np.diff(d.astype(np.int32), axis=2, prepend=0)
    out[f"{name}__depth_rowdiff"] = step.astype(np.int16) if np.abs(step).max() < 2**15 else step
    out[f"{name}__s4"] = arrays["s4"]
    changed = np.flatnonzero(arrays["s5"] != arrays["s4"])
    out[f"{name}__s5_step"] = np.diff(changed, prepend=0).astype(np.int32)
    out[f"{name}__s5_val"] = arrays["s5"].ravel()[changed]
    out[f"{name}__out_sub"] = arrays["out_sub"]
    for k in ("cam_scale", "scale_2_80m"):
        out[f"{name}__{k}"] = arrays[k]
    return out


def load(golden_path):
    """{name: dict(depth, cam_scale, scale_2_80m, <recorded stages>)} from fill_cases.npz"""
    z = np.load(golden_path)
    cases = {}
    for key in z.files:
        if "__" not in key:
            continue
        name, what = key.split("__", 1)
        cases.setdefault(name, {})[what] = z[key]
    for c in cases.values():
        if "depth_rowdiff" in c:
            c["depth"] = np.cumsum(c.pop("depth_rowdiff").astype(np.int64), axis=2)
        c["depth"] = c["depth"].astype(np.float32)
        if "s5_step" in c:
            s5 = c["s4"].copy().ravel()
            s5[np.cumsum(c.pop("s5_step").astype(np.int64))] = c.pop("s5_val")
            c["s5"] = s5.reshape(c["s4"].shape)
    return cases
