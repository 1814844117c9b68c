"""The pose overlay without a GPU: the numpy restatement (tests/vis_ref.py) against the goldens recorded from the
reference (tests/golden/vis_cases.npz), the disc and colour rules against cv2, label_colors against the reference's
get_label_color, the rounding ties the summation order could decide, the argument refusals that need no device, and
compat's routing of Basic_Utils.draw_p2ds on a stand-in class."""
import os
import subprocess
import sys
import types

import numpy as np
import pytest

import vis_ref as V
from pvn3d_b200 import _lib, compat, vis_utils

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "vis_cases.npz")
REF_PY = os.path.join(ROOT, "oracle", "_ref", "py")


@pytest.fixture(scope="module")
def g():
    return dict(np.load(GOLDEN))


def overlay_case(g, i):
    """the inputs of overlay case i: meshes {class: [P,3]} and the rest as recorded"""
    k = f"ov{i}_"
    pts, off = g[k + "mesh_pts"], g[k + "mesh_off"]
    meshes = {c: pts[off[c]:off[c + 1]] for c in range(1, off.size - 1)}
    h, w = (int(x) for x in g[k + "hw"])
    return types.SimpleNamespace(k=k, meshes=meshes, poses=g[k + "poses"], present=g[k + "present"],
                                 order=g[k + "order"], K=g[k + "K"], colors=g[k + "colors"], r=int(g[k + "r"]),
                                 cam_scale=float(g[k + "cam_scale"]), h=h, w=w, seeds=g[k + "seeds"],
                                 name=str(g[k + "name"]))


def frame_images(g, k, h, w):
    """the recorded output frames of case prefix k, rebuilt from their backgrounds and changed pixels; each checked
    against its SHA-256"""
    out, at = [], 0
    for f, seed in enumerate(g[k + "seeds"]):
        n = int(g[k + "chg_cnt"][f])
        img = V.rebuild(V.background(int(seed), h, w), g[k + "chg_idx"][at:at + n], g[k + "chg_val"][at:at + n])
        at += n
        assert V.sha(img) == g[k + "sha"][f].tobytes()
        out.append(img)
    return out


def test_restatement_equals_reference_overlay(g):
    for i in range(int(g["n_overlay"])):
        c = overlay_case(g, i)
        want = frame_images(g, c.k, c.h, c.w)
        drawn = []
        for f, seed in enumerate(c.seeds):
            img, d = V.overlay_frame(V.background(int(seed), c.h, c.w), c.meshes, c.poses[f], c.present[f],
                                     c.order[f], c.K[f], c.colors, c.r, c.cam_scale)
            assert np.array_equal(img, want[f]), (c.name, f)
            drawn += d
        assert [len(p) for p in drawn] == list(g[c.k + "p2ds_cnt"]), c.name
        assert np.array_equal(np.concatenate(drawn), g[c.k + "p2ds"]), c.name


def test_restatement_equals_reference_draw_p2ds(g):
    for i in range(int(g["n_p2ds"])):
        k = f"dp{i}_"
        h, w = (int(x) for x in g[k + "hw"])
        (want,) = frame_images(g, k, h, w)
        p = V.clip(g[k + "p2ds_in"], h, w)
        assert np.array_equal(p, g[k + "p2ds_out"]), k
        img = V.draw(V.background(int(g[k + "seeds"][0]), h, w), p, int(g[k + "r"]), g[k + "color"])
        assert np.array_equal(img, want), k


def test_goldens_cover_the_edges(g):
    radii = {int(g[f"ov{i}_r"]) for i in range(int(g["n_overlay"]))} | {int(g[f"dp{i}_r"]) for i in range(int(g["n_p2ds"]))}
    assert {0, 1, 3, 4, 7} <= radii
    edge = overlay_case(g, 2)
    raw = V.project_raw(V.transform(edge.meshes[1], edge.poses[0, 1]), edge.cam_scale, edge.K[0])
    assert (np.abs(raw) > 2 ** 31).any()                                   # projections beyond int32
    assert np.isnan(edge.poses).any()                                      # a NaN pose
    ins = np.concatenate([g[f"dp{i}_p2ds_in"] for i in range(int(g["n_p2ds"]))])
    assert (ins == -2 ** 31).any() and (ins == 2 ** 31 - 1).any() and (ins < 0).any()
    ycb = overlay_case(g, 0)
    listed = ycb.order[ycb.order > 0]
    assert (ycb.present[np.arange(2)[:, None], ycb.order] == 0)[ycb.order > 0].any()   # a listed class not predicted
    assert len(listed) < ycb.order.size                                                 # zero-padded slots


def test_no_projection_lies_on_a_rounding_tie(g):
    """np.dot may sum the three products in another order than the kernel (BLAS); that can only change a result whose
    quotient lies on a .5 tie.  Count the coordinates within 1e-9 px of one."""
    ties, total = 0, 0
    for i in range(int(g["n_overlay"])):
        c = overlay_case(g, i)
        for f in range(len(c.seeds)):
            for cls in c.order[f]:
                if 1 <= cls < len(c.present[f]) and c.present[f, cls]:
                    raw = V.project_raw(V.transform(c.meshes[cls], c.poses[f, cls]), c.cam_scale, c.K[f])
                    ties += V.near_ties(raw)
                    total += raw.size
    print(f"\nprojected coordinates within 1e-9 px of a .5 tie: {ties} of {total}")
    assert ties == 0


def test_label_colors_match_the_restatement():
    for n_obj in (22, 16, 2):
        want = np.array([V.cv_color(V.label_color(c, n_obj)) for c in range(30)])
        assert np.array_equal(vis_utils.label_colors(30, n_obj), want)
    assert vis_utils.label_colors(22).dtype == np.uint8


def test_cv_color_matches_the_restatement():
    for col in [(255, 0, 0), (300.6, -3, 2.5), (0.5, 1.5, 254.5, 99), (2.5,), (1e10, float("nan"), -7.5),
                (-1e10, 3e9, 2147483647.4), (255.5, 127.5, -0.5), np.array([3, 4, 5], np.uint8)]:
        assert vis_utils.cv_color(col) == tuple(int(v) for v in V.cv_color(col)), col


def test_disc_and_colour_rules_equal_cv2():
    cv2 = pytest.importorskip("cv2")
    for r in list(range(0, 65)) + [97, 128, 199, 256, 300]:
        img = np.zeros((2 * r + 9, 2 * r + 9, 3), np.uint8)
        cv2.circle(img, (r + 4, r + 4), r, (1, 2, 3), -1)
        want = np.zeros_like(img)
        d = V.disc(r)
        want[d[:, 1] + r + 4, d[:, 0] + r + 4] = (1, 2, 3)
        assert np.array_equal(img, want), r
    for (x, y, r) in [(0, 0, 5), (30, 20, 1), (30, 20, 6), (29, 19, 3), (-3, 10, 4)]:   # cut by the borders
        img = np.zeros((20, 30, 3), np.uint8)
        cv2.circle(img, (x, y), r, (9, 9, 9), -1)
        assert np.array_equal(img, V.draw(np.zeros((20, 30, 3), np.uint8), np.array([[x, y]]), r, (9, 9, 9))), (x, y, r)
    for col in [(300.6, -3, 2.5), (0.5, 1.5, 254.5, 99), (2.5,), (1e10, float("nan"), -7.5), (-1e10, 3e9, 2147483647.4)]:
        img = np.zeros((3, 3, 3), np.uint8)
        cv2.circle(img, (1, 1), 0, col, -1)
        assert tuple(img[1, 1]) == vis_utils.cv_color(col), col


def test_label_colors_equal_reference_get_label_color():
    if not os.path.isdir(os.path.join(REF_PY, "lib")):
        pytest.skip("the reference Python is not staged under oracle/_ref/py")
    pytest.importorskip("cv2")
    # a fresh interpreter: the reference's modules stay out of this one
    code = ("import sys, types, json; sys.path.insert(0, %r); from pvn3d_b200 import compat; "
            "compat.install(%r); import numpy as np\n"
            "if not hasattr(np, 'bool'): np.bool = bool\n"
            "from lib.utils.basic_utils import Basic_Utils\n"
            "bu = Basic_Utils(types.SimpleNamespace(dataset_name='linemod'))\n"
            "print(json.dumps([[bu.get_label_color(c, n_obj=n, mode=1) for c in range(30)] for n in (22, 16)]))"
            % (ROOT, REF_PY))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT)
    if r.returncode != 0:
        pytest.skip(f"the staged reference is not importable here: {r.stderr.strip().splitlines()[-1:]}")
    import json

    for n_obj, rows in zip((22, 16), json.loads(r.stdout.strip().splitlines()[-1])):
        want = np.array([vis_utils.cv_color(c) for c in rows], np.uint8)
        assert np.array_equal(vis_utils.label_colors(30, n_obj), want), n_obj


def test_draw_p2ds_refusals_before_any_device_work():
    img = np.zeros((4, 5, 3), np.uint8)
    p = np.zeros((3, 2), np.int32)
    with pytest.raises(TypeError):
        vis_utils.draw_p2ds(img.astype(np.float32), p)
    with pytest.raises(TypeError):
        vis_utils.draw_p2ds(np.zeros((5, 4, 3), np.uint8).transpose(1, 0, 2), p)
    with pytest.raises(TypeError):
        vis_utils.draw_p2ds(img, p.astype(np.float64))
    with pytest.raises(TypeError):
        vis_utils.draw_p2ds(img, np.zeros((3, 3), np.int32))
    with pytest.raises(ValueError):
        vis_utils.draw_p2ds(img, p, r=-1)
    with pytest.raises(ValueError):
        vis_utils.draw_p2ds(img, p, r=1.5)
    with pytest.raises(ValueError):
        vis_utils.draw_p2ds(img, p, color="red")
    q = np.zeros((0, 2), np.int32)
    assert vis_utils.draw_p2ds(img, q) is img                  # nothing to draw: no device needed


def test_c_abi_refusals_before_any_cuda_call():
    lib = _lib.load()
    assert lib.pvn3d_vis_workspace_bytes(2, 480, 640) == 2 * 480 * 640 * 4
    assert lib.pvn3d_vis_workspace_bytes(0, 480, 640) == 0
    fake = 1 << 20                                              # never dereferenced: every call below is refused first
    ws = lib.pvn3d_vis_workspace_bytes(1, 48, 64)
    p2 = lib.pvn3d_vis_draw_p2ds
    assert p2(None, 48, 64, fake, 3, 1, 0, fake, ws, None) == -1
    assert p2(fake, 48, 64, fake, 3, -1, 0, fake, ws, None) == -1
    assert p2(fake, 48, 64, None, 3, 1, 0, fake, ws, None) == -1
    assert p2(fake, 48, 64, fake, 3, 1, 1 << 24, fake, ws, None) == -1
    assert p2(fake, 48, 64, fake, 3, 40000, 0, fake, ws, None) == -2
    assert p2(fake, 48, 64, fake, 3, 1, 0, fake + 4, ws, None) == -1          # workspace not 256-byte aligned
    assert p2(fake, 48, 64, fake, 3, 1, 0, fake, ws - 1, None) == -4
    assert p2(fake, 48, 64, fake, 0, 1, 0, None, 0, None) == 0                 # nothing to draw
    dp = lib.pvn3d_vis_draw_poses
    args = [fake, 1, 48, 64, fake, fake, 3, 10, fake, 0, fake, fake, 2, fake, 1.0, fake, 1, fake, ws, None]

    def rc(**kw):
        a = list(args)
        names = ["img", "b", "h", "w", "pts", "off", "n_cls", "max_pts", "poses", "f64", "present", "order", "s", "k",
                 "cam_scale", "colors", "r", "ws", "ws_bytes", "stream"]
        for k, v in kw.items():
            a[names.index(k)] = v
        return dp(*a)

    assert rc(img=None) == -1 and rc(poses=None) == -1 and rc(order=None) == -1 and rc(k=None) == -1
    assert rc(r=-1) == -1 and rc(n_cls=1) == -1 and rc(s=0) == -1 and rc(f64=2) == -1 and rc(b=0) == -1
    assert rc(r=40000) == -2 and rc(b=70000) == -2 and rc(s=70000) == -2
    assert rc(ws_bytes=ws - 4) == -4


class _StandIn:
    """a class with the reference's draw_p2ds signature; records the calls it runs itself"""
    calls = []

    def draw_p2ds(self, img, p2ds, r=1, color=(255, 0, 0)):
        _StandIn.calls.append((img, p2ds, r, color))
        return "reference"


def test_compat_routes_draw_p2ds(monkeypatch):
    taken = []
    monkeypatch.setattr(vis_utils, "draw_p2ds", lambda img, p2ds, r=1, color=(255, 0, 0): taken.append(r) or img)
    monkeypatch.setattr(vis_utils.torch.cuda, "is_available", lambda: True)
    cls = type("Basic_Utils", (_StandIn,), {})
    before = cls()                                              # an instance made before the patch picks it up
    compat.patch_draw_p2ds(cls)
    orig = cls.draw_p2ds._pvn3d_b200_orig
    compat.patch_draw_p2ds(cls)                                 # idempotent
    assert cls.draw_p2ds._pvn3d_b200_orig is orig
    img = np.zeros((6, 7, 3), np.uint8)
    p = np.zeros((4, 2), np.int32)
    assert before.draw_p2ds(img, p) is img and taken == [1]
    assert before.draw_p2ds(img, p.astype(np.int64), 3, (1.5, 2)) is img and taken == [1, 3]
    _StandIn.calls.clear()
    others = [(img[:, ::-1], p, 1, (1, 2, 3)), (img.astype(np.float32), p, 1, (1, 2, 3)),
              (np.zeros((6, 7, 4), np.uint8), p, 1, (1, 2, 3)), (img, p.astype(np.float64), 1, (1, 2, 3)),
              (img, p.astype(np.int16), 1, (1, 2, 3)), (img, np.zeros((4, 3), np.int32), 1, (1, 2, 3)),
              (img, p, 1.0, (1, 2, 3)), (img, p, -1, (1, 2, 3)), (img, p, True, (1, 2, 3)),
              (img, p, 1, (1, 2, 3, 4, 5)), (img, p, 1, "red"), (img, list(p), 1, (1, 2, 3))]
    for a in others:
        assert before.draw_p2ds(*a) == "reference"
    assert len(_StandIn.calls) == len(others) and taken == [1, 3]
    monkeypatch.setattr(vis_utils.torch.cuda, "is_available", lambda: False)
    assert before.draw_p2ds(img, p) == "reference"              # no CUDA device: the reference's own method


def test_compat_install_patch_vis_rebinds_the_class(monkeypatch):
    mod = types.ModuleType("lib.utils.basic_utils")
    mod.Basic_Utils = type("Basic_Utils", (_StandIn,), {})
    for name in ("lib", "lib.utils"):
        monkeypatch.setitem(sys.modules, name, sys.modules.get(name) or types.ModuleType(name))
    monkeypatch.setitem(sys.modules, "lib.utils.basic_utils", mod)
    monkeypatch.setitem(sys.modules, "lib.pointnet2_utils._ext", None)        # install() binds it; undone afterwards
    monkeypatch.setattr(compat, "install_import_shims", lambda: None)
    compat.install(None)
    assert getattr(mod.Basic_Utils.draw_p2ds, "_pvn3d_b200_orig", None) is None   # off by default
    compat.install(None, patch_vis=True)
    assert mod.Basic_Utils.draw_p2ds._pvn3d_b200_orig is _StandIn.draw_p2ds
