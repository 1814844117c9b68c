"""The numpy restatement of the raster contract (tests/render_ref.py) against an independent float64 ray caster, on
coverage cases with pixel centres exactly on shared edges, an axis-aligned square with analytically known pixels and
the back-projection of its depth; every mutant of the restatement fails at least one of these checks.  Also the
host side of pvn3d_b200.render: mesh packing and load_ply."""
import numpy as np
import pytest

import render_ref as R
from pvn3d_b200.render import load_ply, pack_meshes

H, W = 60, 80
K_SMALL = np.array([[110.0, 0.0, 40.3], [0.0, 112.5, 29.7], [0.0, 0.0, 1.0]])
# m: snapping moves a vertex by at most 1/512 px (~4 um laterally at 0.4 m); on the sphere's grazing faces that moves
# the surface along the ray by up to ~30 um.  Float32 rounding of the depth adds < 0.1 um.
DEPTH_BOUND = 1e-4
MUTANTS = {"centre+0.5": dict(centre=0.5), "no top-left": dict(top_left=False), "affine colour": dict(perspective=False),
           "higher wins ties": dict(low_wins=False), "float edges, no snap": dict(snap=False)}


def _scene():
    """a tilted quad with strongly varying depth (class 1), a small noisy icosphere (class 2), and class 3 = the
    icosphere again at the same pose (an exact tie with class 2)"""
    rng = np.random.default_rng(5)
    quad = (np.array([[-0.2, -0.15, 0], [0.2, -0.15, 0], [0.2, 0.15, 0], [-0.2, 0.15, 0]], np.float32),
            np.array([[0, 1, 2], [0, 2, 3]], np.int32),
            np.array([[255, 0, 0], [0, 255, 0], [0, 0, 255], [250, 250, 10]], np.uint8))
    sph = R.icosphere(1, 0.05, rng, noise=0.05)
    meshes = {1: quad, 2: sph, 3: sph}
    poses = np.stack([np.zeros((3, 4)), R.pose(1.0, 0.2, 0.1, (0.0, 0.0, 0.6)),
                      R.pose(0.3, -0.5, 0.2, (-0.08, 0.03, 0.4)), R.pose(0.3, -0.5, 0.2, (-0.08, 0.03, 0.4))])[None]
    present = np.array([[0, 1, 1, 1]], np.uint8)
    return pack_meshes(meshes), poses, present


def _ideal_check(kw):
    (vtx, col, faces, vo, fo), poses, present = _scene()
    rgb, dpt, lab, _ = R.raster(vtx, col, faces, vo, fo, poses, present, K_SMALL, H, W, **kw)
    c, d, l, e = R.ideal(vtx, col, faces, vo, fo, poses, present, K_SMALL, H, W)
    far = e > 1.0 / 256
    ok_lab = np.array_equal(lab[far], l[far])
    cov = far & (l > 0)
    ok_dpt = bool(np.all(np.abs(dpt[cov].astype(np.float64) - d[cov]) <= DEPTH_BOUND))
    ok_rgb = bool(np.all(np.abs(rgb[cov].astype(np.float64) - c[cov]) <= 1.0))
    return ok_lab, ok_dpt, ok_rgb, int(cov.sum())


def test_restatement_agrees_with_ideal():
    ok_lab, ok_dpt, ok_rgb, n = _ideal_check({})
    assert n > 500
    assert ok_lab and ok_dpt and ok_rgb


def _screen_meshes(polys):
    """triangles given in pixels, placed at z = 2 with identity pose and K = diag(64, 64, 1), cx = cy = 0, so that
    screen position = 32 * (x, y) exactly"""
    verts, faces = [], []
    for tri in polys:
        base = len(verts)
        verts += [(px / 32.0, py / 32.0, 0.0) for px, py in tri]
        faces.append((base, base + 1, base + 2))
    v = np.array(verts, np.float32)
    return {1: (v, np.array(faces, np.int32), np.zeros_like(v, dtype=np.uint8))}


K_SCREEN = np.array([[64.0, 0, 0], [0, 64.0, 0], [0, 0, 1]])
POSE_SCREEN = np.stack([np.zeros((3, 4)), R.pose(0, 0, 0, (0, 0, 2.0))])[None]


def _cover_counts(polys, h=48, w=64, **kw):
    vtx, col, faces, vo, fo = pack_meshes(_screen_meshes(polys))
    *_, fr = R.raster(vtx, col, faces, vo, fo, POSE_SCREEN, np.array([[0, 1]]), K_SCREEN, h, w, frags=True, **kw)
    pix, _ = fr[0]
    return np.bincount(pix, minlength=h * w).reshape(h, w)


def _inside_poly(poly, h, w):
    """pixel centres inside a convex polygon of positive area, with the top-left rule on its boundary"""
    vv, uu = np.mgrid[0:h, 0:w]
    inside = np.ones((h, w), bool)
    n = len(poly)
    for i in range(n):
        (ax, ay), (bx, by) = poly[i], poly[(i + 1) % n]
        e = (bx - ax) * (vv - ay) - (by - ay) * (uu - ax)
        own = (by - ay < 0) or (by == ay and bx - ax > 0)
        inside &= (e > 0) | ((e == 0) & own)
    return inside


SQUARE = [(10, 8), (10, 40), (50, 40), (50, 8)]                    # outlines listed with negative area
FAN_C = (30, 20)
FAN = [(6, 4), (6, 20), (6, 44), (30, 44), (58, 44), (58, 28), (58, 4), (30, 4)]


def _split_square():
    a, b, c, d = SQUARE
    return [(a, b, c), (a, c, d)]


def _fan():
    return [(FAN_C, FAN[i], FAN[(i + 1) % len(FAN)]) for i in range(len(FAN))]


def _coverage_ok(**kw):
    ok = True
    for polys, outline in ((_split_square(), SQUARE), (_fan(), FAN)):
        cnt = _cover_counts(polys, **kw)
        want = _inside_poly(outline[::-1], 48, 64)
        ok &= bool(cnt.max() <= 1) and np.array_equal(cnt == 1, want)
    return ok


def test_shared_edges_cover_once():
    # the diagonal and the fan's spokes pass exactly through pixel centres
    for polys in (_split_square(), _fan()):
        cnt = _cover_counts(polys)
        assert cnt.max() == 1
    assert _coverage_ok()


def _square_ok(**kw):
    """a 0.2 m square facing the camera at 1 m, K = (500, 500, 320, 240): its edges land on pixel centres 270 / 370
    and 190 / 290; the top-left rule keeps columns 270..369 and rows 190..289"""
    v = np.array([[-0.1, -0.1, 0], [0.1, -0.1, 0], [0.1, 0.1, 0], [-0.1, 0.1, 0]], np.float32)
    m = {1: (v, np.array([[0, 1, 2], [0, 2, 3]], np.int32), np.full((4, 3), 200, np.uint8))}
    vtx, col, faces, vo, fo = pack_meshes(m)
    poses = np.stack([np.zeros((3, 4)), R.pose(0, 0, 0, (0, 0, 1.0))])[None]
    k = np.array([[500.0, 0, 320], [0, 500.0, 240], [0, 0, 1]])
    _, dpt, lab, _ = R.raster(vtx, col, faces, vo, fo, poses, np.array([[0, 1]]), k, 480, 640, **kw)
    want = np.zeros((480, 640), bool)
    want[190:290, 270:370] = True
    return np.array_equal(lab[0] == 1, want) and bool(np.all(dpt[0][want] == 1.0))


def test_axis_aligned_square_covers_expected_pixels():
    assert _square_ok()


def _backprojection_ok(**kw):
    """dpt_2_cld (float32, cam_scale 1) of the tilted quad's depth lands on its posed plane"""
    (vtx, col, faces, vo, fo), poses, present = _scene()
    present = np.array([[0, 1, 0, 0]], np.uint8)
    _, dpt, lab, face = R.raster(vtx, col, faces, vo, fo, poses, present, K_SMALL, H, W, **kw)
    vv, uu = np.nonzero(lab[0] == 1)
    d = dpt[0, vv, uu]
    k = K_SMALL.astype(np.float32)
    x = (uu.astype(np.float32) - k[0, 2]) * d / k[0, 0]
    y = (vv.astype(np.float32) - k[1, 2]) * d / k[1, 1]
    pts = np.stack([x, y, d], 1).astype(np.float64)
    dist = R.plane_distance(pts, vtx, faces, face[0, vv, uu], np.repeat(poses[0, 1][None], len(vv), 0))
    bound = d * (np.sqrt(2) / (512 * 110.0) + 2.0 ** -20)
    return len(vv) > 300 and bool(np.all(dist <= bound))


def test_depth_backprojects_onto_surface():
    assert _backprojection_ok()


@pytest.mark.parametrize("name", sorted(MUTANTS))
def test_each_mutant_fails_a_check(name):
    kw = MUTANTS[name]
    ok_lab, ok_dpt, ok_rgb, _ = _ideal_check(kw)
    results = {"ideal labels": ok_lab, "ideal depth": ok_dpt, "ideal colour": ok_rgb,
               "coverage": _coverage_ok(**kw), "square": _square_ok(**kw), "back-projection": _backprojection_ok(**kw)}
    assert not all(results.values()), (name, results)


def test_skipped_triangles():
    # zero area, a vertex behind z_near and a vertex outside the guard band draw nothing; the remaining one draws
    v = np.array([[0, 0, 0], [1, 1, 0], [2, 2, 0],                   # collinear: zero area
                  [0, 0, 0], [0.1, 0, -0.9995], [0, 0.1, 0],          # one vertex at z = 5e-4 < 1e-3
                  [0, 0, 0], [40, 0, 0], [0, 0.1, 0],                 # x = 40 m at 1 m: 20000 px, off the band
                  [-0.02, -0.02, 0], [0.02, -0.02, 0], [0, 0.02, 0]], np.float32)
    m = {1: (v, np.arange(12, dtype=np.int32).reshape(4, 3), np.full((12, 3), 9, np.uint8))}
    vtx, col, faces, vo, fo = pack_meshes(m)
    poses = np.stack([np.zeros((3, 4)), R.pose(0, 0, 0, (0, 0, 1.0))])[None]
    _, dpt, lab, face = R.raster(vtx, col, faces, vo, fo, poses, np.array([[0, 1]]), R.LM_K, 480, 640)
    assert set(np.unique(face[0])) == {-1, 3}


def test_pack_meshes():
    rng = np.random.default_rng(1)
    a, b = R.box(0.05, 2, rng), R.icosphere(1, 0.04, rng)
    vtx, col, faces, vo, fo = pack_meshes({3: b, 1: a})
    assert vo.tolist() == [0, 0, len(a[0]), len(a[0]), len(a[0]) + len(b[0])]
    assert fo.tolist() == [0, 0, len(a[1]), len(a[1]), len(a[1]) + len(b[1])]
    assert np.array_equal(faces[fo[3]:], b[1] + vo[3]) and np.array_equal(col[vo[3]:], b[2])
    same = pack_meshes([None, a, None, b])
    assert all(np.array_equal(x, y) for x, y in zip(same, (vtx, col, faces, vo, fo)))
    with pytest.raises(ValueError):
        pack_meshes({1: (a[0], a[1] + 1000, a[2])})
    with pytest.raises(ValueError):
        pack_meshes({1: (a[0], a[1], a[2][:-1])})
    with pytest.raises(ValueError):
        pack_meshes({1: (a[0], a[1], a[2].astype(np.int32))})
    with pytest.raises(ValueError):
        pack_meshes({256: a})
    with pytest.raises(ValueError):
        pack_meshes({0: a})                                          # class 0 is the background: nothing to draw


def _write_ply(path, v, f, c, fmt, extra=True):
    props = ["property float x", "property float y", "property float z"]
    if extra:
        props += ["property float nx", "property float ny", "property float nz"]
    if c is not None:
        props += ["property uchar red", "property uchar green", "property uchar blue"]
    head = ["ply", f"format {fmt} 1.0", "comment made by a test", f"element vertex {len(v)}", *props,
            f"element face {len(f)}", "property list uchar int vertex_indices", "end_header"]
    with open(path, "wb") as fh:
        fh.write(("\n".join(head) + "\n").encode())
        if fmt == "ascii":
            for i, p in enumerate(v):
                row = [repr(float(x)) for x in p] + (["0", "0", "1"] if extra else [])
                row += [str(int(x)) for x in c[i]] if c is not None else []
                fh.write((" ".join(row) + "\n").encode())
            for t in f:
                fh.write(("3 " + " ".join(str(int(x)) for x in t) + "\n").encode())
        else:
            fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")] + ([("n", "<f4", (3,))] if extra else [])
            fields += [("c", "u1", (3,))] if c is not None else []
            rec = np.zeros(len(v), fields)
            rec["x"], rec["y"], rec["z"] = v[:, 0], v[:, 1], v[:, 2]
            if c is not None:
                rec["c"] = c
            fh.write(rec.tobytes())
            fr = np.zeros(len(f), [("n", "u1"), ("i", "<i4", (3,))])
            fr["n"], fr["i"] = 3, f
            fh.write(fr.tobytes())


@pytest.mark.parametrize("fmt", ["ascii", "binary_little_endian"])
def test_load_ply(tmp_path, fmt):
    v, f, c = R.icosphere(1, 40.0, np.random.default_rng(2))          # millimetres, as LineMOD's models
    p = str(tmp_path / "m.ply")
    _write_ply(p, v, f, c, fmt)
    gv, gf, gc = load_ply(p)
    assert gv.dtype == np.float32 and gf.dtype == np.int32 and gc.dtype == np.uint8
    assert np.array_equal(gv, v) and np.array_equal(gf, f) and np.array_equal(gc, c)
    _write_ply(p, v, f, None, fmt, extra=False)
    gv, gf, gc = load_ply(p)
    assert np.array_equal(gv, v) and not gc.any()


def test_load_ply_refuses(tmp_path):
    p = str(tmp_path / "bad.ply")
    v, f, c = R.icosphere(0, 1.0, np.random.default_rng(3))
    _write_ply(p, v, f, c, "binary_big_endian")
    with pytest.raises(ValueError):
        load_ply(p)
    _write_ply(p, v, f, c, "ascii")
    txt = open(p).read().replace("3 0 ", "4 0 9 ", 1)                # a quad
    open(p, "w").write(txt)
    with pytest.raises(ValueError):
        load_ply(p)
    open(p, "w").write("not a ply\n")
    with pytest.raises(ValueError):
        load_ply(p)
