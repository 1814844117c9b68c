"""The render edge cases (tests/render_edge_cases.py) on the host: each reaches what it claims, counted from the
restatement's own per-slot candidate counts (the kernel's scan input); the restatement agrees with the float64 ray
caster on the new geometry; and each wrong reference gives a different frame from the restatement on the case named
for it, so the bit-exact GPU comparison rejects it."""
import numpy as np
import pytest

import render_edge_cases as E
import render_ref as R

# test_render_host's bounds: pixels more than 1/256 px from a projected edge, depth within 1e-4 m, colour within 1
EDGE_PX, DEPTH_BOUND = 1.0 / 256, 1e-4


def _blocks(counts):
    """(scan blocks, the blocks holding a slot with candidate pixels)"""
    flat = counts.reshape(-1)
    return -(-flat.size // E.SCAN_BLOCK), set(np.unique(np.nonzero(flat)[0] // E.SCAN_BLOCK).tolist())


def _first_fragment(counts):
    """the scan's exclusive offset of every slot: the index of the slot's first fragment"""
    flat = counts.reshape(-1)
    return np.cumsum(flat) - flat


def test_bench_shape_passes_block_1024():
    case = E.bench()
    counts = case.counts()
    n_faces = case.packed[2].shape[0]
    nb, drawn = _blocks(counts)
    assert n_faces == 4 * 99372 and case.b == 32 and (case.h, case.w) == (480, 640)
    assert nb == 12422 and nb > E.SCAN_BLOCK                             # 13 passes of the block-total scan
    assert 3 * n_faces >= E.SCAN_BLOCK * E.SCAN_BLOCK                    # frames 3.. lie wholly past block 1024
    assert len([blk for blk in drawn if blk > E.SCAN_BLOCK]) > 5000
    per_frame = counts.sum(1)
    assert (per_frame > 0).all()
    assert (case.present.sum(1)[:16] == 1).all() and (case.present.sum(1)[16:] == 4).all()   # render, fuse


DRAWN_BLOCKS = {"1024": {0}, "1025": {0, 1}, "1024^2": set(range(0, 1024, 64)), "1024^2+1": {0, 1024},
                "1024^2+1023": {0, 1024}, "last block only": {1025}}


@pytest.mark.parametrize("variant", sorted(E.SCAN_VARIANTS))
def test_scan_boundaries(variant):
    case = E.scan(variant)
    slots = case.b * case.packed[2].shape[0]
    want_slots = {"1024": 1024, "1025": 1025, "1024^2": 1024 ** 2, "1024^2+1": 1024 ** 2 + 1,
                  "1024^2+1023": 1024 ** 2 + 1023, "last block only": 1025 * 1024 + 80}[variant]
    assert slots == want_slots
    nb, drawn = _blocks(case.counts())
    assert nb == E.SCAN_BLOCKS[variant]
    assert drawn == DRAWN_BLOCKS[variant], sorted(drawn)[:8]


def test_over_2e32_fragments():
    case, rgb, dpt, lab = E.over_2e32()
    counts = case.counts()[0]
    hw = E.BIG * E.BIG
    assert counts.sum() > 2 ** 32, counts.sum()
    fo = case.packed[4]
    half, *tie = case.visible
    full = np.ones(counts.size, bool)
    full[fo[half]:fo[half + 1]] = False
    assert (counts[full] == hw).all() and (counts[~full] == hw // 2).all()   # candidate boxes: the whole frame
    first = _first_fragment(counts)
    for c in case.visible:                                              # what is visible lies past 2^32
        assert first[fo[c]] >= 2 ** 32, c
    depth = case.poses[0, 1:, 2, 3]
    assert np.array_equal(depth.astype(np.float32).astype(np.float64), depth)   # exact float32 depths
    assert depth[tie[0] - 1] == depth[tie[1] - 1] and len(np.unique(depth)) == depth.size - 1
    assert depth.argmin() + 1 == half and tie[0] < tie[1]
    assert set(np.unique(lab).tolist()) == {half, tie[0]} and (lab[0, :, :2048] == tie[0]).all()
    assert dpt.dtype == np.float32 and rgb.dtype == np.uint8


def test_over_2e32_tie_is_by_class():
    # the analytic frame's rule on a small copy the restatement can hold: the same two tied quads, and the half quad
    # whose left edge lies on a pixel column, at 1/64 of the size
    case, _, _, lab = E.over_2e32()
    half, *tie = case.visible
    keep = [half, *tie]
    s = 1 / 64
    K = E.BIG_K.copy()
    K[:2] *= s
    present = np.zeros_like(case.present)
    present[0, keep] = 1
    small = R.raster(*case.packed, case.poses, present, K, 64, 64)
    want = np.full((64, 64), tie[0])
    want[:, 32:] = half
    assert np.array_equal(small[2][0], want)


def test_guard_and_near_boundaries():
    case = E.guard()
    vtx, _, _, vo, _ = case.packed
    flags = {}
    for f in range(case.b):
        sx, _, ok, _, q = R._vertices(vtx, vo, case.poses[f], case.K[f], case.z_near)
        flags[f] = sx, ok, q[2]
    sx, ok, _ = flags[0]
    assert sx[vo[1]] == 16384.0 and ok[vo[1]]                            # on the band: usable
    assert 16384.0 < sx[vo[2]] <= 16384.0 + 2.0 ** -9 and not ok[vo[2]]  # a float32 ulp beyond
    sx, ok, _ = flags[1]
    assert sx[vo[1]] == np.nextafter(16384.0, np.inf) and not ok[vo[1]]  # a float64 ulp beyond
    _, ok, z = flags[2]
    assert z[vo[3]] == case.z_near and ok[vo[3]]                         # on the near plane: usable
    assert z[vo[4]] == case.z_near - 2.0 ** -25 and not ok[vo[4]]
    rgb, dpt, lab, face = case.want()
    assert set(np.unique(lab[0]).tolist()) == {0, 1} and not lab[1].any()
    assert set(np.unique(lab[2]).tolist()) == {0, 3} and set(np.unique(lab[3]).tolist()) == {5, 6}
    s = R.faces_setup(vtx, case.packed[2], vo, case.packed[4], case.poses[3], case.present[3], case.K[3], case.h,
                      case.w, case.z_near)
    assert s["area"].size == 2 and (s["area"] > 2 ** 45).all() and (s["area"] < 2 ** 47).all()
    assert np.abs(np.concatenate([s["X"], s["Y"]])).max() >= 16000 * 256


def test_tiny_frame_chunks_span_frames():
    case = E.tiny_frames()
    counts = case.counts()
    frame_of = np.repeat(np.arange(case.b), counts.sum(1))
    starts = np.arange(0, frame_of.size, E.CHUNK)
    ends = np.minimum(starts + E.CHUNK, frame_of.size) - 1
    spans = frame_of[ends] - frame_of[starts] + 1
    assert frame_of.size > 20 * E.CHUNK and spans.min() >= 2 and spans.max() >= 20, (frame_of.size, spans.min())


def _ideal_ok(case, poses, present, K):
    """test_render_host's comparison with the ray caster, its bounds taken per pixel.  The 1e-4 m depth bound is
    test_render_host's for fx = 110 at about 0.4 m; the snap's depth error grows as z^2 / f, so the bound does too
    past those.  The colour is compared on triangles at least 2 px tall: on smaller ones the 1/512 px snap moves
    the barycentrics by more than a level."""
    K = np.broadcast_to(K, (len(poses), 3, 3))
    rgb, dpt, lab, face = R.raster(*case.packed, poses, present, K, case.h, case.w, case.z_near)
    c, d, l, e = R.ideal(*case.packed, poses, present, K, case.h, case.w, case.z_near)
    vtx, _, faces, vo, _ = case.packed
    tall = np.zeros(lab.shape, bool)
    for f in range(len(poses)):
        sx, sy, *_ = R._vertices(vtx, vo, poses[f], K[f], case.z_near)
        p = np.stack([sx, sy], -1)[faces[face[f][face[f] >= 0]]]          # [n,3,2] the winners' vertices
        e0, e1, e2 = p[:, 1] - p[:, 0], p[:, 2] - p[:, 1], p[:, 0] - p[:, 2]
        area2 = np.abs(e0[:, 0] * e2[:, 1] - e0[:, 1] * e2[:, 0])
        longest = np.sqrt(np.maximum.reduce([(x * x).sum(1) for x in (e0, e1, e2)]))
        tall[f][face[f] >= 0] = area2 / longest >= 2.0
    far = e > EDGE_PX
    cov = far & (l > 0)
    bound = (DEPTH_BOUND * np.maximum(1.0, 110.0 / np.minimum(K[:, 0, 0], K[:, 1, 1]))[:, None, None]
             * np.maximum(1.0, (d / 0.4) ** 2))
    assert np.array_equal(lab[far], l[far])
    assert np.all(np.abs(dpt.astype(np.float64) - d)[cov] <= bound[cov])
    assert np.all(np.abs(rgb.astype(np.float64) - c)[cov & tall] <= 1.0)
    return int(cov.sum()), int((cov & tall).sum())


@pytest.mark.parametrize("name", ["guard", "per-frame K", "1x1", "1x4096", "4096x1", "7x5", "tiny frames"])
def test_restatement_agrees_with_ideal(name):
    if name == "guard":
        # frame 3's two triangles one at a time: where they cross in depth the snap decides, not the ray caster
        case = E.guard()
        pr = np.concatenate([case.present, case.present[3:]])
        pr[3, 6] = pr[4, 5] = 0
        n = _ideal_ok(case, case.poses[[0, 1, 2, 3, 3]], pr, case.K[[0, 1, 2, 3, 3]])
    elif name == "per-frame K":
        case = E.per_frame_k(scale=0.125)
        n = _ideal_ok(case, case.poses, case.present, case.K)
    elif name == "tiny frames":
        case = E.tiny_frames()
        n = _ideal_ok(case, case.poses[:64], case.present[:64], case.K)
    else:
        case = E.frame_size(*map(int, name.split("x")))
        n = _ideal_ok(case, case.poses, case.present, case.K)
    assert n[0] > 0


def _differs(a, b):
    return not (np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))
                and np.array_equal(a[2], b[2]))


WRONG = ["guard band one ulp narrower", "guard band one ulp wider", "z_near compared with >", "frame 0's K for all",
         "K[0,1] read", "higher face wins ties"]


@pytest.mark.parametrize("name", WRONG)
def test_wrong_reference_differs(name, monkeypatch):
    if name == "higher face wins ties":
        case = E.contention()
        right, wrong = case.want(), case.want(low_wins=False)
    elif name in ("frame 0's K for all", "K[0,1] read"):
        case = E.per_frame_k()
        right = case.want()
        if name == "K[0,1] read":
            monkeypatch.setattr(R, "_vertices", E.vertices_mutant(skew=True))
            wrong = case.want()
        else:
            wrong = case.want(K=case.K[0])
    else:
        case = E.guard()
        right = case.want()
        if name == "z_near compared with >":
            monkeypatch.setattr(R, "_vertices", E.vertices_mutant(near_strict=True))
        else:
            monkeypatch.setattr(R, "GUARD", np.nextafter(16384.0, 0.0 if "narrower" in name else np.inf))
        wrong = case.want()
    assert _differs(right, wrong), f"{name}: the {case.name} case does not tell it from the restatement"


def test_class_layouts():
    case = E.classes()
    assert case.packed[3].size == 257
    assert all(np.array_equal(a, b) for a, b in zip(case.packed, E.classes(as_list=True).packed))
    fo, vo = case.packed[4], case.packed[3]
    assert fo[78] == fo[77] and vo[78] > vo[77]                          # class 77: vertices, no faces
    assert (np.diff(fo) == 0).sum() == 256 - 3                           # runs of empty classes
    _, _, lab, _ = case.want()
    assert set(np.unique(lab[0]).tolist()) == {0, 1, 128}                # class 1 wins every tie with 255
    assert set(np.unique(lab[1]).tolist()) == {0, 255} and set(np.unique(lab[2]).tolist()) == {0, 128}
    assert not lab[3].any()


def test_foreign_faces_are_skipped():
    case = E.foreign_faces()
    vtx, _, faces, vo, fo = case.packed
    cls_f = np.repeat(np.arange(3), np.diff(fo))
    own = (faces >= vo[cls_f][:, None]) & (faces < vo[cls_f + 1][:, None])
    assert own.all(1).tolist() == [True, True, False, False, False, False]
    assert faces.min() < 0 and faces.max() >= len(vtx)
    face = case.want()[3]
    assert set(np.unique(face[0]).tolist()) == {-1, 0, 1} and set(np.unique(face[1]).tolist()) == {-1, 1}
    # drawn, the foreign faces would show: face 2 uses class 1's vertex 0 at class 2's pose
    loose = R.raster(vtx, case.packed[1], faces, np.array([0, 0, 0, 6], np.int32), fo, case.poses, case.present,
                     case.K, case.h, case.w)[3]
    assert (loose[0] >= 2).any()


def test_poses():
    case = E.poses()
    p = case.poses
    assert np.isnan(p[0, 2]).all() and np.isinf(p[0, 3]).all() and not case.present[0, 2:].any()
    assert np.isnan(p[1, 2]).any() and np.isinf(p[1, 3]).any() and case.present[1, 2:].all()
    assert p[2, 1, 2, 3] < 0 and np.linalg.det(p[3, 1, :, :3]) < 0 and np.linalg.det(p[3, 2, :, :3]) < 0
    _, _, lab, _ = case.want()
    assert set(np.unique(lab[0]).tolist()) == {0, 1} and set(np.unique(lab[1]).tolist()) == {0, 1}
    assert set(np.unique(lab[2]).tolist()) == {0, 2}
    assert (lab[3] == 1).sum() > 500 and (lab[3] == 2).sum() > 100 and not np.array_equal(lab[3], lab[4])


def test_contention():
    case = E.contention()
    fo = case.packed[4]
    assert fo[-1] == 11500 and case.counts().sum() > 10 ** 5
    rgb, dpt, lab, face = case.want()
    cov = lab[0] > 0
    assert cov.sum() > 1600 and set(np.unique(lab[0]).tolist()) == {0, 1, 2}
    assert np.ptp(dpt[0][cov].view(np.int32)) < 400                      # within a few hundred float32 steps
