"""Edge cases of csrc/render.cu, built for the bit-exact comparison with the restatement (tests/render_ref.py).

Each builder returns a `Case`: the meshes (what MeshRenderer takes) and their packing, the pose table, the present
flags, K, the frame size, z_near and what the case claims to exercise.  The host tests (test_render_edges_host.py)
show from the restatement's own per-slot candidate counts that each case reaches what it claims; the GPU tests
(test_render_edges_gpu.py) compare the kernel with the restatement, or with the analytic frame of `over_2e32`.

`vertices_mutant` and the keyword mutants of `R.raster` are the wrong references each case must tell apart.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

import render_ref as R
from pvn3d_b200 import synth
from pvn3d_b200.render import pack_meshes

SCAN_BLOCK = 1024          # kScanBlock: faces per block of the two-level scan
CHUNK = 1024               # kChunk: fragments per CTA step of the fragment pass
F32_ULP_OUT = float(np.nextafter(np.float32(1.0), np.float32(2.0)))


@dataclass
class Case:
    name: str
    claim: str
    meshes: object             # {class id: (vtx, faces, colors)} or a list; None: the packing only (C ABI)
    packed: tuple              # pack_meshes(meshes): vtx, col, faces, vtx_off, face_off
    poses: np.ndarray          # [B,n_cls,3,4] float64, float32-representable where a test passes float32
    present: np.ndarray        # [B,n_cls] uint8
    K: np.ndarray              # [3,3] or [B,3,3] float64
    h: int
    w: int
    z_near: float = 1e-3
    background: tuple | None = None

    @property
    def b(self):
        return self.poses.shape[0]

    def want(self, poses=None, K=None, **kw):
        """the restatement's (rgb, depth, labels, face) of the case; poses / K replace the case's own"""
        return R.raster(*self.packed, self.poses if poses is None else poses, self.present,
                        self.K if K is None else K, self.h, self.w, self.z_near, self.background, **kw)

    def counts(self):
        """[B, n_faces] candidate-pixel counts of the kernel's scan slots"""
        vtx, _, faces, vo, fo = self.packed
        return R.slot_counts(vtx, faces, vo, fo, self.poses, self.present, self.K, self.h, self.w, self.z_near)


def _case(name, claim, meshes, poses, present, K, h, w, **kw):
    return Case(name, claim, meshes, pack_meshes(meshes), np.asarray(poses, np.float64),
                np.asarray(present, np.uint8), np.asarray(K, np.float64), h, w, **kw)


def _k(fx, fy, cx, cy):
    return np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])


def _f32(p):
    return np.asarray(p, np.float32).astype(np.float64)


def _rand_pose(rng, xy, z):
    return _f32(R.pose(*rng.uniform(-np.pi, np.pi, 3), (rng.uniform(-xy, xy), rng.uniform(-xy, xy), rng.uniform(*z))))


def _flat(v, f, rgb):
    """one mesh of the given vertices [V,3] and faces, every vertex coloured rgb"""
    v = np.asarray(v, np.float32)
    return v, np.asarray(f, np.int32).reshape(-1, 3), np.tile(np.asarray(rgb, np.uint8), (len(v), 1))


IDENTITY = np.concatenate([np.eye(3), np.zeros((3, 1))], 1)


def _at(t):
    p = IDENTITY.copy()
    p[:, 3] = t
    return p


# ---- 1. the benchmark's shape -------------------------------------------------------------------------------------
def bench(b=32):
    """tools/render_bench.py's largest shape: 4 classes of 99,372-face boxes, 32 frames of 480x640.  Frames 0-15 are
    render frames (one class each), 16-31 fuse frames (all four).  b * n_faces = 12.7 M slots, 12,422 scan blocks:
    13 passes of the block-total scan, and frames 3 on lie wholly past block 1024."""
    rng = np.random.default_rng(21)
    meshes = {c: R.box(np.array([0.06, 0.05, 0.04]) * s, 91, rng) for c, s in zip(range(1, 5), (1.0, 0.8, 1.2, 0.9))}
    poses = np.zeros((b, 5, 3, 4))
    present = np.zeros((b, 5), np.uint8)
    for f in range(b):
        for c in ([1 + f % 4] if f < b // 2 else range(1, 5)):
            poses[f, c] = _rand_pose(rng, 0.12, (0.5, 1.0))
            present[f, c] = 1
    return _case("bench", "more than 1024 scan blocks; render and fuse frames past block 1024", meshes, poses,
                 present, R.LM_K, 480, 640)


# ---- 2. exact scan boundaries -------------------------------------------------------------------------------------
SCAN_VARIANTS = {
    # name: (frames, [(kind, faces)] in class order)
    "1024": (1, [("sphere", 80), ("undrawn", 944)]),
    "1025": (1, [("sphere", 80), ("zero", 944), ("tri", 1)]),
    "1024^2": (16, [("sphere", 80), ("undrawn", 65456)]),
    "1024^2+1": (1, [("sphere", 80), ("zero", 1024 * 1024 - 80), ("tri", 1)]),
    "1024^2+1023": (1, [("sphere", 80), ("zero", 1024 * 1024 + 1023 - 160), ("sphere", 80)]),
    "last block only": (1, [("undrawn", 1025 * 1024), ("sphere", 80)]),
}
SCAN_BLOCKS = {"1024": 1, "1025": 2, "1024^2": 1024, "1024^2+1": 1025, "1024^2+1023": 1025, "last block only": 1026}


def scan(variant):
    """b * n_faces on and just past the scan's block and pass boundaries.  Padding faces take slots and draw nothing:
    an undrawn class, or a drawn class of collinear (zero-area) faces."""
    frames, layout = SCAN_VARIANTS[variant]
    rng = np.random.default_rng(31)
    sph = R.icosphere(1, 0.03, rng, noise=0.05)
    meshes = {}
    poses = np.zeros((frames, len(layout) + 1, 3, 4))
    present = np.zeros((frames, len(layout) + 1), np.uint8)
    for c, (kind, n) in enumerate(layout, 1):
        if kind == "sphere":
            meshes[c] = sph
        elif kind == "tri":
            meshes[c] = _flat([[-0.02, -0.02, 0], [0.03, -0.01, 0], [0, 0.025, 0]], [0, 1, 2], (10, 200, 30))
        else:   # a repeated vertex: zero snapped area at any pose (collinear points would not stay so after snapping)
            meshes[c] = _flat([[0, 0, 0], [0.01, 0.01, 0], [0.02, 0.02, 0]], np.tile([0, 1, 1], n), (1, 2, 3))
        assert len(meshes[c][1]) == n
        for f in range(frames):
            poses[f, c] = _f32(R.pose(0.3 * f + c, 0.2 * c, 0.1, (0.02 * (c - 2), 0.01 * f - 0.05, 0.4)))
            present[f, c] = kind != "undrawn"
    return _case(f"scan {variant}", f"{SCAN_BLOCKS[variant]} scan blocks", meshes, poses, present,
                 _k(80.0, 80.0, 32.0, 24.0), 48, 64)


# ---- 3. more than 2^32 fragments ----------------------------------------------------------------------------------
BIG = 4096
BIG_K = _k(4096.0, 4096.0, 2048.0, 2048.0)


def over_2e32(n_quads=255):
    """one 4096x4096 frame of n_quads fronto-parallel quads (classes 1..n_quads), each projecting to about +-6000 px so
    that both its triangles' candidate boxes are the whole frame: about 8.5e9 fragments for 255 quads.  Depths are
    exact float32 values 0.5 + k/1024 in shuffled class order.  The three visible quads all have class ids whose
    fragments lie past 2^32 in scan order: `half` (nearest, its left edge on pixel column 2048, so it covers columns
    2048..4095) and the tie pair `tie` (next nearest, equal depth), of which the lower class must win columns 0..2047.
    Returns (case, expected rgb, depth, labels) with the analytic frame."""
    rng = np.random.default_rng(41)
    classes = np.arange(1, n_quads + 1)
    half, tie = n_quads - 3, (n_quads - 9, n_quads - 1)
    rank = np.full(n_quads + 1, -1)
    rank[half], rank[tie[0]], rank[tie[1]] = 0, 1, 1
    rest = [c for c in classes if rank[c] < 0]
    rank[rest] = 2 + rng.permutation(len(rest))
    depth = 0.5 + rank / 1024.0
    colors = rng.integers(0, 256, (n_quads + 1, 3), dtype=np.uint8)
    meshes, poses = {}, np.zeros((1, n_quads + 1, 3, 4))
    for c in classes:
        r = 6000.0 * depth[c] / BIG_K[0, 0]
        x0 = 0.0 if c == half else -r
        meshes[int(c)] = _flat([[x0, -r, 0], [r, -r, 0], [r, r, 0], [x0, r, 0]], [[0, 1, 2], [0, 2, 3]], colors[c])
        poses[0, c] = _at((0.0, 0.0, depth[c]))
    present = np.ones((1, n_quads + 1), np.uint8)
    want_lab = np.full((1, BIG, BIG), min(tie), np.uint8)
    want_lab[:, :, BIG // 2:] = half
    want_dpt = depth[want_lab].astype(np.float32)
    want_rgb = colors[want_lab]
    case = _case(f"over 2^32 ({n_quads} quads)", "a fragment total above 2^32; the visible quads past it", meshes,
                 poses, present, BIG_K, BIG, BIG)
    case.visible = (half, *tie)
    return case, want_rgb, want_dpt, want_lab


# ---- 4. guard band and near plane at their boundaries -------------------------------------------------------------
GUARD_FX = 16384.0
GUARD_FX_OUT = float(np.nextafter(GUARD_FX, np.inf))
NEAR = 0.5
NEAR_IN_Z = -0.25                                                       # camera z = -0.25 + 0.75 = 0.5 exactly
NEAR_OUT_Z = float(np.nextafter(np.float32(NEAR_IN_Z), np.float32(-1.0)))   # one float32 ulp nearer: 0.5 - 2^-25


def guard():
    """frame 0: K with fx = 16384, cx = 0 puts class 1's vertex (1, 0, 1) at sx = 16384.0 exactly (usable) and class
    2's vertex (1 + 2^-23, ...) one float32 ulp beyond (skipped); frame 1: fx one float64 ulp above 16384 moves class
    1's vertex just outside the band (skipped); frame 2: z_near = 0.5 with class 3's vertex at camera z 0.5 exactly
    (usable) and class 4's a float32 ulp nearer (skipped); frame 3: classes 5 and 6, two triangles in depth whose
    vertices project to +-16000 px, so the snapped area and the edge functions come near 2^47."""
    y1, y2 = 1.0 / 1024, 2.7 / 1024
    m = {
        1: _flat([[1, 0, 1], [0, -y1, 1], [0, y1, 1]], [0, 1, 2], (200, 40, 40)),
        2: _flat([[F32_ULP_OUT, -y2, 1], [0, -y2 - y1, 1], [0, -y2 + y1, 1]], [0, 1, 2], (40, 200, 40)),
        3: (np.array([[0.05, 0, NEAR_IN_Z], [-0.05, -0.1, 0], [-0.05, 0.1, 0]], np.float32), np.array([[0, 1, 2]]),
            np.array([[255, 0, 0], [0, 255, 0], [0, 0, 255]], np.uint8)),
        4: (np.array([[0.05, 0.2, NEAR_OUT_Z], [-0.05, 0.1, 0], [-0.05, 0.3, 0]], np.float32), np.array([[0, 1, 2]]),
            np.array([[255, 255, 0], [0, 255, 255], [255, 0, 255]], np.uint8)),
    }
    k_wide = _k(100.0, 100.0, 32.0, 64.0)
    # class 5 / 6 vertices at given screen positions (px) and camera depths; object = camera coordinates
    def at_px(pts):
        return [[(sx - k_wide[0, 2]) * z / k_wide[0, 0], (sy - k_wide[1, 2]) * z / k_wide[1, 1], z] for sx, sy, z in pts]
    rng = np.random.default_rng(51)
    m[5] = (np.array(at_px([(-16000, -15900, 1.0), (16000, -3000, 1.6), (-2000, 16000, 0.8)]), np.float32),
            np.array([[0, 1, 2]]), rng.integers(0, 256, (3, 3), dtype=np.uint8))
    # class 6 faces the camera at 1.0395 m; class 5 runs from 1.038 to 1.041 m across the frame, so they cross in it
    m[6] = (np.array(at_px([(15900, 16000, 1.0395), (-16000, 2000, 1.0395), (3000, -16000, 1.0395)]), np.float32),
            np.array([[0, 1, 2]]), rng.integers(0, 256, (3, 3), dtype=np.uint8))
    poses = np.zeros((4, 7, 3, 4))
    present = np.zeros((4, 7), np.uint8)
    for f, cls in ((0, (1, 2)), (1, (1, 2)), (2, (3, 4)), (3, (5, 6))):
        for c in cls:
            poses[f, c] = _at((0.0, 0.0, 0.75)) if c in (3, 4) else IDENTITY
            present[f, c] = 1
    K = np.stack([_k(GUARD_FX, GUARD_FX, 0.0, 64.0), _k(GUARD_FX_OUT, GUARD_FX, 0.0, 64.0), k_wide, k_wide])
    return _case("guard", "vertices on both sides of the guard band and the near plane; edge functions near 2^47",
                 m, poses, present, K, 128, 64, z_near=NEAR)


# ---- 5. per-frame intrinsics --------------------------------------------------------------------------------------
def per_frame_k(scale=1.0):
    """eight frames of the same two objects under eight K: LineMOD's, YCB's, fx != fy, a principal point outside the
    frame, nonzero K[0,1], K[1,0] and row 2 (not read), a short and a long focal length, fractional centres.  scale
    shrinks K and the frame together (the ray-cast reference runs at 1/8)."""
    rng = np.random.default_rng(61)
    meshes = {1: R.icosphere(3, 0.05, rng, noise=0.04), 2: R.box(np.array([0.04, 0.03, 0.05]), 6, rng)}
    ks = [R.LM_K, synth.K_YCB1, _k(450.0, 700.0, 320.0, 240.0), _k(572.0, 573.0, -150.0, 700.0),
          np.array([[572.4, 30.0, 325.0], [12.0, 573.6, 242.0], [0.05, -0.02, 1.7]]), _k(150.0, 150.0, 320.5, 239.5),
          _k(2500.0, 2500.0, 310.0, 250.0), _k(600.25, 599.5, 319.75, 240.125)]
    K = np.stack(ks).astype(np.float64)
    K[:, :2] *= scale
    h, w = int(round(480 * scale)), int(round(640 * scale))
    poses = np.zeros((8, 3, 3, 4))
    present = np.zeros((8, 3), np.uint8)
    for f, k in enumerate(ks):
        z = 3.0 if f == 6 else 0.6
        # aim the objects at pixel (w/2 +- 40, h/2) of the full-size frame under this K
        for c, du in ((1, -40.0), (2, 40.0)):
            x = (320.0 + du - k[0, 2]) * z / k[0, 0]
            y = (240.0 - k[1, 2]) * z / k[1, 1]
            poses[f, c] = _f32(R.pose(*rng.uniform(-np.pi, np.pi, 3), (x, y, z)))
            present[f, c] = 1
    return _case("per-frame K", "eight different K, one per frame", meshes, poses, present, K, h, w)


# ---- 6. frame sizes -----------------------------------------------------------------------------------------------
SIZES = [(1, 1), (1, 4096), (4096, 1), (7, 5), (481, 641), (4096, 4096)]


def frame_size(h, w):
    """one ordinary object (plus a box in front of it) centred near the frame's middle; for 1-pixel-wide frames the
    object spans the frame's length and crosses its sides"""
    rng = np.random.default_rng(71 + h + w)
    level = 3 if h * w >= 4096 * 4096 else 2
    meshes = {1: R.icosphere(level, 0.05, rng, noise=0.05), 2: R.box(np.array([0.02, 0.03, 0.01]), 3, rng)}
    f = max(h, w) * 1.5 if max(h, w) > 8 else 40.0
    K = _k(f, f, (w - 1) / 2 + 0.3, (h - 1) / 2 - 0.2)
    poses = np.stack([[np.zeros((3, 4)), _f32(R.pose(0.3, 0.5, 0.7, (0.004, -0.003, 0.5))),
                       _f32(R.pose(0.1, -0.2, 0.3, (0.01, 0.01, 0.45)))]])
    present = np.array([[0, 1, 1]], np.uint8)
    return _case(f"size {h}x{w}", f"a {h}x{w} frame", meshes, poses, present, K, h, w)


def tiny_frames(b=1024):
    """1024 frames of 3x5, each with the 80-face sphere at its own pose: a 1024-fragment chunk spans several frames"""
    rng = np.random.default_rng(81)
    meshes = {1: R.icosphere(1, 0.05, rng, noise=0.05)}
    poses = np.zeros((b, 2, 3, 4))
    for f in range(b):
        poses[f, 1] = _rand_pose(rng, 0.06, (0.15, 0.3))
    present = np.zeros((b, 2), np.uint8)
    present[:, 1] = 1
    present[::97, 1] = 0                                                # some frames draw nothing
    return _case("tiny frames", "fragment chunks across frames", meshes, poses, present, _k(8.0, 8.0, 2.0, 1.0), 3, 5)


# ---- 7. class layouts ---------------------------------------------------------------------------------------------
def classes(as_list=False):
    """n_cls = 256 with meshes only at classes 1, 128 and 255 (255: the same mesh as 1, so they tie where both are
    drawn at one pose), class 77 with vertices and no faces, and present flags set on classes without a mesh.  Frame 0
    draws 1, 77, 128 and 255; frame 1 only 255 (label 255 through the uint8 cast); frame 2 128 and 77; frame 3
    nothing.  as_list: the same meshes as a list with None entries."""
    rng = np.random.default_rng(91)
    sph = R.icosphere(2, 0.05, rng, noise=0.05)
    bx = R.box(np.array([0.04, 0.05, 0.03]), 4, rng)
    lonely = (rng.uniform(-0.05, 0.05, (7, 3)).astype(np.float32), np.zeros((0, 3), np.int32),
              rng.integers(0, 256, (7, 3), dtype=np.uint8))
    d = {1: sph, 77: lonely, 128: bx, 255: sph}
    meshes = [d.get(c) for c in range(256)] if as_list else d
    poses = np.zeros((4, 256, 3, 4))
    poses[:] = _f32(R.pose(0.2, 0.4, 0.1, (0.0, 0.0, 0.5)))
    poses[:, 128] = _f32(R.pose(0.5, 0.1, 0.9, (0.03, 0.02, 0.45)))
    present = np.zeros((4, 256), np.uint8)
    present[0, [1, 50, 77, 128, 255]] = 1
    present[1, [255, 254, 2]] = 1
    present[2, [77, 128, 0]] = 1
    return _case("classes", "256 classes, sparse ids, label 255, a class without faces", meshes, poses, present,
                 _k(200.0, 200.0, 80.0, 60.0), 120, 160)


def foreign_faces():
    """hand-packed arrays (what pack_meshes refuses): class 2 holds, besides its own triangle, faces that index class
    1's vertices, a negative index and one past the last vertex.  The range rule skips all three."""
    vtx = np.array([[-0.05, -0.05, 0], [0.05, -0.05, 0], [0, 0.05, 0],                     # class 1
                    [-0.02, 0.0, -0.05], [0.06, 0.01, -0.05], [0.01, 0.07, -0.05]], np.float32)   # class 2
    col = np.array([[200, 0, 0], [0, 200, 0], [0, 0, 200], [90, 90, 0], [0, 90, 90], [90, 0, 90]], np.uint8)
    faces = np.array([[0, 1, 2],                                                          # class 1
                      [3, 4, 5], [0, 4, 5], [3, -1, 5], [3, 4, 6 + 7], [2, 1, 0]], np.int32)   # class 2
    vo = np.array([0, 0, 3, 6], np.int32)
    fo = np.array([0, 0, 1, 6], np.int32)
    poses = np.zeros((2, 3, 3, 4))
    poses[:, 1] = poses[:, 2] = _at((0.0, 0.0, 0.5))
    poses[1, 2] = _f32(R.pose(0.0, 0.0, 0.3, (0.01, 0.0, 0.45)))
    present = np.array([[0, 1, 1], [0, 0, 1]], np.uint8)
    return Case("foreign faces", "faces outside their class's vertex range", None, (vtx, col, faces, vo, fo), poses,
                present, _k(300.0, 300.0, 40.0, 30.0), 60, 80)


# ---- 8. poses -----------------------------------------------------------------------------------------------------
MIRROR = np.diag([-1.0, 1.0, 1.0])


def poses():
    """frame 0: NaN and inf poses in absent classes; frame 1: a NaN translation and an inf rotation entry in present
    classes (they draw nothing) beside a normal one; frame 2: an object behind the camera; frame 3: mirrored poses
    (det R = -1: the winding flips); frame 4: frame 3's poses unmirrored."""
    rng = np.random.default_rng(101)
    meshes = {1: R.icosphere(2, 0.05, rng, noise=0.08), 2: R.box(np.array([0.05, 0.03, 0.02]), 3, rng),
              3: R.icosphere(1, 0.03, rng)}
    p = np.zeros((5, 4, 3, 4))
    present = np.zeros((5, 4), np.uint8)
    base = {c: _f32(R.pose(0.3 * c, -0.4 * c, 0.2, (0.04 * (c - 2), 0.01 * c, 0.5 + 0.05 * c))) for c in (1, 2, 3)}
    p[0, 1], present[0, 1] = base[1], 1
    p[0, 2], p[0, 3] = np.nan, np.inf
    p[0, 0] = -np.inf
    p[1, 1], p[1, 2], p[1, 3] = base[1], base[2], base[3]
    p[1, 2, 0, 3] = np.nan
    p[1, 3, 1, 1] = np.inf
    present[1, 1:] = 1
    p[2, 1], p[2, 2] = base[1], base[2]
    p[2, 1, 2, 3] = -0.6                                                 # behind the camera
    present[2, 1:3] = 1
    for c in (1, 2):
        p[3, c], p[4, c] = base[c], base[c]
        p[3, c, :, :3] = MIRROR @ base[c][:, :3]
        present[3, c] = present[4, c] = 1
    return _case("poses", "non-finite, behind-camera and mirrored poses", meshes, p, present,
                 _k(200.0, 200.0, 80.0, 60.0), 120, 160)


# ---- 9. contention ------------------------------------------------------------------------------------------------
def contention(n=10000, n_dup=1500):
    """n small triangles over one 40x40 px region at depths within ~2e-5 of 1 m (about 170 float32 steps, so distinct
    faces tie too), in shuffled face order, plus n_dup duplicates of some of them with their own vertex colours (exact
    depth ties).  The faces are split over classes 1 and 2, so ties fall within a class and across the two."""
    rng = np.random.default_rng(111)
    k = _k(500.0, 500.0, 32.0, 32.0)
    centre = rng.uniform(12, 52, (n, 1, 2))
    px = centre + rng.uniform(-8, 8, (n, 3, 2))
    z = 1.0 + rng.uniform(0, 2e-5, (n, 3))
    v = np.concatenate([(px - k[:2, 2]) * z[..., None] / k[[0, 1], [0, 1]], z[..., None]], -1)     # [n,3,3]
    dup = rng.choice(n, n_dup, replace=False)
    v = np.concatenate([v, v[dup]])
    v = v[rng.permutation(len(v))].astype(np.float32)
    split = len(v) * 3 // 5
    meshes = {}
    for c, part in ((1, v[:split]), (2, v[split:])):
        meshes[c] = (part.reshape(-1, 3), np.arange(part.shape[0] * 3, dtype=np.int32).reshape(-1, 3),
                     rng.integers(0, 256, (part.shape[0] * 3, 3), dtype=np.uint8))
    poses = np.stack([[np.zeros((3, 4)), IDENTITY, IDENTITY]])
    return _case("contention", f"{len(v)} faces over one 40x40 px region, exact depth ties", meshes, poses,
                 np.array([[0, 1, 1]], np.uint8), k, 64, 64)


# ---- wrong references ---------------------------------------------------------------------------------------------
_VERTICES = R._vertices


def vertices_mutant(near_strict=False, skew=False):
    """R._vertices with one rule changed, to be monkeypatched in: q_2 > z_near instead of >=, or sx reading K[0,1]
    as (fx q_0 + K[0,1] q_1) / q_2 + cx"""
    def vertices(vtx, vtx_off, pose_b, k, z_near):
        sx, sy, ok, iz, q = _VERTICES(vtx, vtx_off, pose_b, k, z_near)
        with np.errstate(all="ignore"):
            if skew:
                sx = (k[0, 0] * q[0] + k[0, 1] * q[1]) / q[2] + k[0, 2]
            if near_strict:
                ok = ok & (q[2] > z_near)
            ok = ok & (np.abs(sx) <= R.GUARD)
        return sx, sy, ok, iz, q
    return vertices
