"""Golden vectors of get_item's training augmentation recorded from the REFERENCE ITSELF (build container only).

Imports the unmodified reference ycb_dataset.py and linemod_dataset.py by path (pcl stubbed by
compat.install_import_shims) and calls their rgb_add_noise, gaussian_noise, linear_motion_blur and add_real_back
methods on a stub `self` whose rng replays the draws of an explicit parameter record (so the reference runs exactly
the record's branches) and whose background frame is written to a temporary directory as the PNGs it reads; the
ColorJitter is torchvision's own with get_params returning the record's draws.  While recording it asserts that
tests/augment_ref.py reproduces them and cv2 / PIL:
  * cv2 BGR2HSV / HSV2BGR, PIL convert("L"), PIL RGB<->HSV: bit-equal over all 2^24 inputs;
  * GaussianBlur on a dense sigma sweep and the blur on
    every image case; the motion-blur line's taps for all 360 x 15 (angle, length) pairs;
  * filter2D with the sharpen and motion kernels within 1 of cv2 (the share of differing pixels is logged);
  * ColorJitter, the HSV augmentor, add_real_back bit-equal; gaussian_noise fed the same field bit-equal but for
    float64-vs-float32 truncation ties (logged);
and that every wrong variant of augment_ref.MUTANTS is told apart by at least one recorded case.  Logs the
reference's CPU time per 480x640 frame.  The tests read only the npz.

    python tests/golden/make_golden_augment.py        # writes augment_cases.npz + make_golden_augment.log
"""
import importlib.util
import os
import sys
import tempfile
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
REF = os.environ.get("PVN3D_REFERENCE", "/root/reference/pvn3d")

import cv2  # noqa: E402
import torch  # noqa: E402
import torchvision  # noqa: E402
import torchvision.transforms as transforms  # noqa: E402
from PIL import Image  # noqa: E402

import augment_ref as R  # noqa: E402
from oracle import ext_cpu  # noqa: E402
from pvn3d_b200 import compat  # noqa: E402

compat.install_import_shims()
sys.modules["lib.pointnet2_utils._ext"] = ext_cpu
sys.path.insert(0, REF)
LOG = []


def log(msg):
    print(msg)
    LOG.append(msg)


def load(rel, name):
    cwd = os.getcwd()
    os.chdir(REF)
    try:
        spec = importlib.util.spec_from_file_location(name, os.path.join(REF, "datasets", rel))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        os.chdir(cwd)
    mod.imshow = lambda *a, **k: None       # linemod add_real_back shows its mask
    return mod


class ScriptedRng:
    """numpy.random stand-in that returns a scripted sequence: rand() values, randint() results, randn() fields"""

    def __init__(self, seq):
        self.seq = list(seq)

    def _next(self, kind):
        k, v = self.seq.pop(0)
        assert k == kind, (k, kind)
        return v

    def rand(self):
        return self._next("rand")

    def randint(self, *a):
        return self._next("randint")

    def randn(self, *shape):
        v = self._next("randn")
        assert v.shape == shape
        return v


def script(ps, dataset, field, extra):
    """the rng draws that make the reference's rgb_add_noise run pass record `ps`"""
    yes, no = 0.9, 0.1
    seq = [("rand", 0.5), ("range", float(ps["s_factor"])), ("range", float(ps["v_factor"]))]
    if dataset == R.YCB:
        seq.append(("rand", yes if ps["sharpen"] else no))
        if ps["sharpen"]:
            seq.append(("rand", (ps["sharpen_w"] - 9) / 3))
    seq.append(("rand", yes if ps["motion"] else no))
    if ps["motion"]:
        seq += [("rand", (ps["angle"] + 0.5) / 360), ("rand", (ps["length"] - 1 + 0.5) / 15)]
    seq.append(("rand", yes if ps["gauss"] else no))
    if ps["gauss"]:
        seq += [("rand", 0.5 if ps["ksize"] == 3 else 0.1), ("rand", ps["sigma"])]
    if dataset == R.YCB:
        seq += [("rand", 0.5), ("randint", int(ps["noise_sigma"])), ("randn", field.astype(np.float64)),
                ("rand", yes if ps["extra"] else no)]
    return seq


def exact_scale(ps, dataset):
    """a sharpen weight rand()*3+9 with rand() a multiple of 2^-20, so that the script's (w - 9) / 3 gives it back"""
    u = np.floor((ps["sharpen_w"] - 9) / 3 * 2 ** 20) / 2 ** 20
    ps["sharpen_w"] = u * 3 + 9


class Stub:
    pass


def ref_noise_pass(mod, cls, img, ps, dataset, field, extra):
    st = Stub()
    st.rng = ScriptedRng(script(ps, dataset, field, extra))
    st.rand_range = lambda rng, lo, hi: rng._next("range")       # the record's factor itself
    st.gaussian_noise = lambda rng, im, s: cls.gaussian_noise(st, rng, im, s)
    st.linear_motion_blur = lambda im, a, n: cls.linear_motion_blur(st, im, a, n)
    orig = np.random.normal
    np.random.normal = lambda loc, scale, size: extra.astype(np.float64) * scale
    try:
        out = cls.rgb_add_noise(st, img)
    finally:
        np.random.normal = orig
    assert not st.rng.seq
    return out


def ref_jitter(img, p):
    cj = transforms.ColorJitter(0.2, 0.2, 0.2, 0.05)
    cj.get_params = lambda *a: (torch.tensor(p["order"]), float(p["brightness"]), float(p["contrast"]),
                                float(p["saturation"]), float(p["hue"]))
    return np.array(cj(Image.fromarray(img)))


def ref_add_real_back(mod, cls, dataset, rgb, labels, dpt, back_rgb, back_labels, back_dpt):
    with tempfile.TemporaryDirectory() as root:
        st = Stub()
        st.real_gen = lambda: "000000"
        if dataset == R.YCB:
            st.root = root
            base = os.path.join(root, "000000")
            Image.fromarray(back_dpt.astype(np.uint16)).save(base + "-depth.png")
            Image.fromarray(back_labels).save(base + "-label.png")
            Image.fromarray(back_rgb).save(base + "-color.png")
        else:
            st.cls_root = root
            for d in ("depth", "mask", "rgb"):
                os.makedirs(os.path.join(root, d))
            Image.fromarray(back_dpt.astype(np.uint16)).save(os.path.join(root, "depth", "000000.png"))
            Image.fromarray(back_labels).save(os.path.join(root, "mask", "000000.png"))
            Image.fromarray(back_rgb).save(os.path.join(root, "rgb", "000000.png"))
        msk = dpt > 1e-6
        return cls.add_real_back(st, rgb, labels, dpt.astype(np.uint16), msk)


def exhaustive_checks():
    a = np.arange(256 ** 3, dtype=np.int64)
    px = np.stack([a >> 16, (a >> 8) & 255, a & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    im = Image.fromarray(px)
    checks = {"cv2 BGR2HSV": (R.cv_bgr2hsv(px), cv2.cvtColor(px, cv2.COLOR_BGR2HSV)),
              "cv2 HSV2BGR": (R.cv_hsv2bgr(px), cv2.cvtColor(px, cv2.COLOR_HSV2BGR)),
              "PIL convert('L')": (R.pil_l(px), np.array(im.convert("L"))),
              "PIL RGB->HSV": (R.pil_rgb2hsv(px), np.array(im.convert("HSV"))),
              "PIL HSV->RGB": (R.pil_hsv2rgb(px), np.array(Image.fromarray(px, "HSV").convert("RGB")))}
    for name, (got, want) in checks.items():
        assert np.array_equal(got, want), name
        log(f"{name}: bit-equal over all 2^24 inputs")
    for m in ("hsv2bgr_round",):
        with R.mutant(m):
            assert not np.array_equal(R.cv_hsv2bgr(px), checks["cv2 HSV2BGR"][1])
    # the fixed-point taps are not exposed by cv2: whole blurs of a random image over a dense sweep of sigma
    rng = np.random.default_rng(11)
    img = rng.integers(0, 256, (9, 13, 3), dtype=np.uint8)
    sig = np.concatenate([[0.0, 1e-300, 1e-12, 1e-6], np.linspace(0, 1, 4001)[1:], rng.random(1000)])
    for k in (3, 5):
        for s in sig:
            if k == 5 and s == 0:
                continue
            assert np.array_equal(R.gaussian_blur(img, k, s), cv2.GaussianBlur(img, (k, k), s)), (k, s)
    log(f"GaussianBlur 3x3 / 5x5: bit-equal on a 9x13 image for {len(sig)} sigmas in [0, 1) each (5x5 sigma 0 below)")
    # cv2's 5x5 sigma-0 (binomial 1-4-6-4-1) path gives results that change with the buffer's address on narrow
    # images: compare where it is stable, and log how far it strays on a 9x13 image
    spread = set()
    for off in range(32):
        buf = np.empty(img.size + 32, np.uint8)
        v = buf[off:off + img.size].reshape(img.shape)
        v[...] = img
        spread.add(int(np.abs(R.gaussian_blur(img, 5, 0.0).astype(int) - cv2.GaussianBlur(v, (5, 5), 0.0)).max()))
    big = rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)
    for _ in range(3):
        assert np.array_equal(R.gaussian_blur(big, 5, 0.0), cv2.GaussianBlur(big, (5, 5), 0.0))
    log(f"GaussianBlur 5x5 sigma 0: bit-equal on 480x640 (3 calls); on a 9x13 image cv2 itself varies with the "
        f"buffer's alignment, max |diff| over 32 alignments {sorted(spread)}")
    n = 0
    for ang in range(360):
        for ln in range(1, 16):
            rad = np.deg2rad(ang)
            dx, dy = np.cos(rad), np.sin(rad)
            side = int(max(abs(dx), abs(dy)) * ln * 2)
            got_side, pts = R.motion_line(ang, ln)
            assert got_side == side
            if side <= 0:
                continue
            kern = np.zeros((side, side))
            c = side // 2
            cv2.line(kern, (c, c), tuple(map(int, (dx * ln + c, dy * ln + c))), 1.0)
            mine = np.zeros_like(kern)
            for (y, x) in pts:
                mine[y, x] = 1.0
            assert np.array_equal(mine, kern), (ang, ln)
            n += 1
    log(f"motion-blur line: tap sets equal to cv2.line for all 360 x 15 (angle, length) pairs ({n} non-empty)")


def image_cases(rng):
    """(name, rgb, depth, labels, back_rgb, back_labels, back_depth): ragged sizes, all background, all foreground,
    saturated pixels, every border"""
    out = []
    for name, h, w in (("ragged", 7, 11), ("tiny", 2, 3), ("tall", 31, 4), ("wide", 5, 70), ("frame", 480, 640)):
        rgb = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        rgb[: max(1, h // 5)] = 255
        rgb[-1, :] = 0
        dpt = rng.integers(0, 3000, (h, w)).astype(np.float32)
        dpt[rng.random((h, w)) < 0.3] = 0
        lab = (rng.random((h, w)) < 0.5).astype(np.uint8) * 5
        back = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        bl = (rng.random((h, w)) < 0.3).astype(np.uint8) * 2
        bd = rng.integers(0, 3000, (h, w)).astype(np.float32)
        out.append((name, rgb, dpt, lab, back, bl, bd))
    h, w = 9, 10
    z = np.zeros((h, w), np.uint8)
    base = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    out.append(("all_background", base, np.zeros((h, w), np.float32), z, base[::-1].copy(), z,
                np.full((h, w), 700, np.float32)))
    out.append(("all_foreground", base, np.full((h, w), 500, np.float32), z + 1, base, z + 1,
                np.full((h, w), 700, np.float32)))
    return out


def pass_records(rng, dataset, n):
    p = R.host_draw(rng, dataset, [R.KIND_SYN] * n)
    for f in range(n):
        ps = p[f]["passes"][0]
        ps["motion"] = ps["gauss"] = 1
        ps["sharpen"] = int(dataset == R.YCB)
        ps["extra"] = int(dataset == R.YCB and f % 2 == 0)
        ps["ksize"] = (3, 5)[f % 2]
        ps["sigma"] = (0.0, 0.444, 1e-9, 0.93)[f % 4]      # 0.444: the error diffusion changes a 5x5 tap
        ps["length"] = (1, 15, 6, 3)[f % 4]
        ps["noise_sigma"] = (0, 14, 24, 7)[f % 4] if dataset == R.YCB else 0
        exact_scale(ps, dataset)
    return p


def main():
    ycb = load(os.path.join("ycb", "ycb_dataset.py"), "ref_ycb_dataset")
    lm = load(os.path.join("linemod", "linemod_dataset.py"), "ref_linemod_dataset")
    classes = {R.YCB: (ycb, ycb.YCB_Dataset), R.LINEMOD: (lm, lm.LM_Dataset)}
    log(f"cv2 {cv2.__version__}, PIL {Image.__version__}, torchvision {torchvision.__version__}, numpy {np.__version__}")
    exhaustive_checks()
    rng = np.random.default_rng(2026)
    out = {}
    told = {m: [] for m in R.MUTANTS}
    cases = image_cases(rng)
    for dataset in (R.YCB, R.LINEMOD):
        mod, cls = classes[dataset]
        recs = pass_records(rng, dataset, len(cases))
        jrec = R.host_draw(rng, dataset, [R.KIND_REAL] * len(cases))
        for i, (name, rgb, dpt, lab, back, bl, bd) in enumerate(cases):
            key = f"{dataset}_{name}"
            if dataset == R.LINEMOD and name == "ragged":
                bl = np.repeat(bl[..., None], 3, -1)
                bl[..., 1] = 0                                         # a 3-channel mask, channels differ
            h, w = rgb.shape[:2]
            field = rng.standard_normal((h, w, 3)).astype(np.float32)
            extra = rng.standard_normal((h, w, 3)).astype(np.float32)
            ps = recs[i]["passes"][0]
            # the jitter
            jr = jrec[i]
            want_j = ref_jitter(rgb, jr)
            got_j = R.color_jitter(rgb, jr)
            assert np.array_equal(got_j, want_j), key
            # one noise pass, step by step
            want_hsv = ref_noise_pass(mod, cls, rgb, _only(ps, "hsv"), dataset, np.zeros_like(field),
                                      np.zeros_like(extra))
            assert np.array_equal(R.hsv_scale(rgb, ps["s_factor"], ps["v_factor"]), want_hsv), key
            want_gauss = cv2.GaussianBlur(rgb, (int(ps["ksize"]),) * 2, float(ps["sigma"]))
            assert np.array_equal(R.gaussian_blur(rgb, int(ps["ksize"]), float(ps["sigma"])), want_gauss), key
            fk = {"sharpen": R.sharpen_kernel(ps["sharpen_w"]), "motion": R.motion_kernel(ps["angle"], ps["length"])}
            f2d = {}
            for kname, kern in fk.items():
                if kern is None:
                    continue
                want = cv2.filter2D(rgb, -1, kern)
                got = R.filter2d(rgb, kern)
                diff = np.abs(got.astype(int) - want)
                assert diff.max() <= 1, (key, kname)
                f2d[kname] = want
                log(f"  {key}: filter2D {kname} {kern.shape[0]}x{kern.shape[1]}: {(diff > 0).mean():.2e} of values "
                    f"differ by 1 from cv2")
            want_pass = ref_noise_pass(mod, cls, rgb, ps, dataset, field, extra)
            got_pass = R.noise_pass(rgb, ps, dataset, field, extra)
            dp = np.abs(got_pass.astype(int) - want_pass)
            assert dp.max() <= 1, key
            # the composite (channel order of the network: the reference's add_real_back gets the image as it is)
            want_rgb, want_dpt = ref_add_real_back(mod, cls, dataset, want_pass, lab, dpt, back, bl, bd)
            got_rgb, got_dpt = R.add_real_back(want_pass, lab, dpt, back, bl, bd, dataset)
            assert np.array_equal(got_rgb, want_rgb) and np.array_equal(got_dpt, want_dpt.astype(np.float32)), key
            log(f"  {key} {h}x{w}: jitter order {[int(o) for o in jr['order']]}, HSV, GaussianBlur k{int(ps['ksize'])} "
                f"sigma {float(ps['sigma']):.3g}, add_real_back bit-equal; whole pass (motion length "
                f"{int(ps['length'])}, noise sigma {int(ps['noise_sigma'])}, extra {int(ps['extra'])}): "
                f"{(dp > 0).mean():.2e} of values differ by 1")
            rec = {"rgb": rgb, "depth": dpt, "labels": lab, "back_rgb": back, "back_labels": bl, "back_depth": bd,
                   "field": field, "extra": extra, "record": recs[i:i + 1].view(np.uint8),
                   "jrecord": jrec[i:i + 1].view(np.uint8), "jitter": want_j, "hsv": want_hsv, "gauss": want_gauss,
                   "pass": want_pass, "out_rgb": want_rgb, "out_depth": want_dpt.astype(np.float32)}
            for kname, v in f2d.items():
                rec["f2d_" + kname] = v
            if name == "frame":      # keep the npz small: the big frame only checks the restatement here
                rec = {k: v for k, v in rec.items() if k in ("record", "jrecord")}
            for k, v in rec.items():
                out[f"{key}/{k}"] = v
            for m in R.MUTANTS:
                with R.mutant(m):
                    bad = (not np.array_equal(R.color_jitter(rgb, jr), want_j)
                           or not np.array_equal(R.hsv_scale(rgb, ps["s_factor"], ps["v_factor"]), want_hsv)
                           or not np.array_equal(R.gaussian_blur(rgb, int(ps["ksize"]), float(ps["sigma"])),
                                                 want_gauss)
                           or np.abs(R.noise_pass(rgb, ps, dataset, field, extra).astype(int) - want_pass).max() > 1
                           or not all(np.array_equal(a, b) for a, b in
                                      zip(R.add_real_back(want_pass, lab, dpt, back, bl, bd, dataset),
                                          (want_rgb, want_dpt.astype(np.float32)))))
                if bad and name != "frame":
                    told[m].append(key)
    for m, keys in told.items():
        assert keys, f"mutant {m} is not told apart by any case"
        log(f"mutant {m}: rejected by {', '.join(keys)}")
    # the reference's CPU time per 480x640 frame
    mod, cls = classes[R.YCB]
    name, rgb, dpt, lab, back, bl, bd = next(c for c in cases if c[0] == "frame")
    ps = R.host_draw(np.random.default_rng(1), R.YCB, [R.KIND_SYN])[0]["passes"][0]
    exact_scale(ps, R.YCB)
    field = np.random.default_rng(2).standard_normal((480, 640, 3))
    ts = []
    for _ in range(10):
        t0 = time.perf_counter()
        ref_jitter(rgb, R.host_draw(np.random.default_rng(3), R.YCB, [R.KIND_REAL])[0])
        x = ref_noise_pass(mod, cls, rgb, ps, R.YCB, field, field)
        ref_add_real_back(mod, cls, R.YCB, x, lab, dpt, back, bl, bd)
        ts.append(time.perf_counter() - t0)
    log(f"reference YCB syn frame on the CPU (ColorJitter + rgb_add_noise + add_real_back, which here also writes the background PNGs it reads; cv2 "
        f"{cv2.getNumThreads()} threads, {os.cpu_count()} cpus): 480x640 median {np.median(ts) * 1e3:.1f} ms, "
        f"min {min(ts) * 1e3:.1f} ms over 10 calls")
    path = os.path.join(HERE, "augment_cases.npz")
    np.savez_compressed(path, **out)
    log(f"wrote augment_cases.npz ({os.path.getsize(path)} bytes): restatement == reference on every case")
    with open(os.path.join(HERE, "make_golden_augment.log"), "w") as f:
        f.write("\n".join(LOG) + "\n")


def _only(ps, what):
    """a copy of pass `ps` that runs only the HSV augmentor (and no noise)"""
    q = ps.copy()
    q["sharpen"] = q["motion"] = q["gauss"] = q["extra"] = 0
    q["noise_sigma"] = 0
    return q


if __name__ == "__main__":
    main()
