"""The numpy restatement of get_item's augmentation (tests/augment_ref.py) against the goldens recorded from the
reference and cv2 / PIL / torchvision (tests/golden/make_golden_augment.py); every wrong variant of
augment_ref.MUTANTS is told apart by at least one case; the C ABI's refusals before any launch.  No GPU needed."""
import os

import numpy as np
import pytest

import augment_ref as R
from pvn3d_b200 import _lib

CASES = [f"{d}_{n}" for d in ("ycb", "linemod")
         for n in ("ragged", "tiny", "tall", "wide", "all_background", "all_foreground")]


@pytest.fixture(scope="module")
def cases(golden_dir):
    z = np.load(os.path.join(golden_dir, "augment_cases.npz"))
    out = {}
    for k in z.files:
        case, field = k.split("/")
        out.setdefault(case, {})[field] = z[k]
    return out


def _rec(raw):
    return raw.view(R.PARAMS_DTYPE)[0]


def _check(c, dataset):
    """True when the restatement (under the current mutant) reproduces every recorded output of case c"""
    p, jr = _rec(c["record"]), _rec(c["jrecord"])
    ps = p["passes"][0]
    rgb = c["rgb"]
    ok = np.array_equal(R.color_jitter(rgb, jr), c["jitter"])
    ok &= np.array_equal(R.hsv_scale(rgb, ps["s_factor"], ps["v_factor"]), c["hsv"])
    ok &= np.array_equal(R.gaussian_blur(rgb, int(ps["ksize"]), float(ps["sigma"])), c["gauss"])
    for name, kern in (("sharpen", R.sharpen_kernel(ps["sharpen_w"])),
                       ("motion", R.motion_kernel(int(ps["angle"]), int(ps["length"])))):
        if "f2d_" + name in c:
            ok &= int(np.abs(R.filter2d(rgb, kern).astype(int) - c["f2d_" + name]).max()) <= 1
    got = R.noise_pass(rgb, ps, dataset, c["field"], c["extra"])
    ok &= int(np.abs(got.astype(int) - c["pass"]).max()) <= 1
    out_rgb, out_dpt = R.add_real_back(c["pass"], c["labels"], c["depth"], c["back_rgb"], c["back_labels"],
                                       c["back_depth"], dataset)
    ok &= np.array_equal(out_rgb, c["out_rgb"]) and np.array_equal(out_dpt, c["out_depth"])
    return bool(ok)


def test_goldens_hold_every_case(cases):
    assert set(CASES) <= set(cases)


@pytest.mark.parametrize("name", CASES)
def test_restatement_matches_reference_goldens(cases, name):
    assert _check(cases[name], name.split("_")[0])


def test_every_mutant_is_told_apart_by_some_golden(cases):
    for m in R.MUTANTS:
        with R.mutant(m):
            told = [n for n in CASES if not _check(cases[n], n.split("_")[0])]
        assert told, m


def test_records_layout():
    assert R.PARAMS_DTYPE.itemsize == 208 and R.PASS_DTYPE.itemsize == 80
    assert R.PARAMS_DTYPE.fields["passes"][1] == 48


def test_host_draw_structure():
    rng = np.random.default_rng(0)
    p = R.host_draw(rng, R.LINEMOD, [R.KIND_REAL, R.KIND_RENDER, R.KIND_FUSE] * 50)
    assert (p["jitter"] == np.tile([1, 0, 0], 50)).all()
    assert (p["back"] == np.tile([0, 1, 0], 50)).all()
    assert (p["passes"]["sharpen"] == 0).all() and (p["passes"]["noise_sigma"] == 0).all()


def test_abi_refuses_bad_arguments():
    lib = _lib.load()
    assert lib.pvn3d_augment_workspace_bytes(0, 480, 640) == 0
    assert lib.pvn3d_augment_workspace_bytes(4, 480, 640) >= 2 * 4 * 480 * 640 * 3
    assert lib.pvn3d_augment_workspace_bytes(60000, 4000, 4000) == 0            # 64-bit indexing
    args = [1] * 7 + [1, 2, 8, 8, 0, 1, 1, 0, 0, 1, 1 << 20, 0]
    for i in range(7):                                                       # null inputs
        a = list(args)
        a[i] = None if i != 5 else 2                                         # back_label_channels 2
        assert lib.pvn3d_augment_apply(*a) == -1
    bad_ds = list(args)
    bad_ds[11] = 2
    assert lib.pvn3d_augment_apply(*bad_ds) == -1
    assert lib.pvn3d_augment_draw(1, None, 4, 0, 1, None) == -1
    assert lib.pvn3d_augment_draw(1, 1, 4, 5, 1, None) == -1
    assert lib.pvn3d_augment_probe(8, 1, 4, 1, None) == -1
