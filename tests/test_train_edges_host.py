"""Without a GPU: the edge cases of tests/train_edge_cases.py hit the edges they are named for, their shared-memory
constants are csrc/train.cu's, and each bound of tests/test_train_edges_gpu.py rejects every mutant of
tests/train_ref.py in float64 on the CPU -- so a kernel that computed a mutant could not pass the GPU tests."""
import os
import re

import numpy as np
import pytest
import torch

import train_edge_cases as E
import train_ref as R

TRAIN_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pvn3d_b200", "csrc", "train.cu")


def _cu():
    with open(TRAIN_CU) as f:
        return f.read()


def _const(src, name):
    m = re.search(rf"constexpr int {name} = ([0-9* ]+);", src)
    assert m, f"{name} not found in train.cu"
    return eval(m.group(1))          # noqa: S307 -- an integer product such as 48 * 1024


def test_footprints_follow_the_kernel_layout():
    src = _cu()
    assert _const(src, "kLossTile") == E.TILE and _const(src, "kLossMaxKp") == E.KP_MAX
    assert _const(src, "kLossMaxClasses") == E.C_MAX and _const(src, "kTgtThreads") == E.TGT_THREADS
    assert _const(src, "kTgtMaxSmem") == E.TGT_MAX_SMEM
    # the staged layouts and the static arrays the footprints are computed from
    assert "static_cast<size_t>(a->n_cls) * (kLossTile + 1) * sizeof(float)" in src
    assert "static_cast<size_t>(kLossTile) * (a->n_kp * 3 + 1) * sizeof(float)" in src
    assert "__shared__ float s_red[kLossWarps * kLossMaxKp];" in src and "__shared__ int s_cnt[kLossWarps];" in src
    assert E.STATIC_SMEM == 784 and E.NO_OPT_IN_DYNAMIC == 48368


def test_c94_and_c95_exceed_the_limit_without_the_opt_in():
    between = [c for c in range(1, E.C_MAX + 1) if E.NO_OPT_IN_DYNAMIC < E.seg_smem(c) <= E.SMEM_LIMIT]
    assert between == [94, 95], between
    assert not [k for k in range(1, E.KP_MAX + 1) if E.NO_OPT_IN_DYNAMIC < E.of_smem(k) <= E.SMEM_LIMIT]
    # the cases sit on both sides of both limits
    assert E.seg_smem(31) <= E.NO_OPT_IN_DYNAMIC and E.seg_smem(96) > E.SMEM_LIMIT
    assert E.of_smem(31) <= E.NO_OPT_IN_DYNAMIC and E.of_smem(32) > E.SMEM_LIMIT
    assert {31, 94, 95, 96} <= set(E.FOCAL_C) and set(E.FRESH_C) == {94, 95, 96} and set(E.FRESH_K) == {31, 32}
    assert {31, 32} <= set(E.OF_K) and E.KP_MAX in E.OF_K and E.C_MAX in E.FOCAL_C


def test_cases_hit_the_tile_edges():
    # focal rows and OF points: several tiles with a ragged last one
    assert any(m > E.TILE and m % E.TILE for m in E.FOCAL_M) and 1 in E.FOCAL_M
    assert {n % E.TILE for n in E.OF_N} >= {0, 1, E.TILE - 1} and max(E.OF_N) > 90 * E.TILE
    # NCHW: every HW either puts several images in one tile or crosses a tile boundary inside an image
    for hw in E.NCHW_HW:
        shapes = [s for s in E.NCHW_SHAPES[:-2] if s[2] * s[3] == hw]
        assert {s[0] for s in shapes} == set(E.NCHW_N)
        several = any(E.tile_images(hw, s[0] * hw).max() >= 2 for s in shapes)
        crosses = hw > E.TILE and hw % E.TILE != 0
        assert several or crosses, hw
    assert E.tile_images(100, 300).max() == 2 and E.tile_images(1, 5).max() == 5
    # PVN3DLoss: focal tiles straddle frames, and some straddle an ok and a not-ok frame
    rows = E.PVN_B * E.PVN_N
    starts = np.arange(0, rows, E.TILE)
    f0, f1 = starts // E.PVN_N, np.minimum(starts + E.TILE, rows - 1) // E.PVN_N
    ok = np.asarray(E.PVN_OK)
    assert (ok[f0] != ok[f1]).sum() >= 2
    # OF: frames with no and with every labelled point
    _, _, lab = E.of_case(5, E.TILE + 1, 2, seed=0)
    assert (lab[0] == 0).all() and (lab[-1] > 0).all() and (lab[1:, -1] > 0).all()
    _, _, flab = E.of_nonfinite_case(seed=3)
    assert {np.float32(1e-9), np.float32(2e-8)} <= set(flab.reshape(-1).tolist())


def test_target_cases_hold_ids_int32_cannot():
    _, labels, ids, _, _, _ = E.targets_case(4, 600, 22, 8, 22, seed=1, wide=True)
    i32 = np.iinfo(np.int32)
    for a in (labels, ids):
        wide = (a < i32.min) | (a > i32.max)
        assert wide.any()
        # their int32 truncation lands on real classes: a wrapping conversion would give those points offsets
        assert ((a[wide].astype(np.int32) >= 1) & (a[wide].astype(np.int32) < 22)).any()
    assert E.tgt_smem(*E.TGT_FULL) == E.TGT_MAX_SMEM and E.TGT_FULL[2] <= 4096
    assert E.tgt_smem(E.TGT_FULL[0], E.TGT_FULL[1], E.TGT_FULL[2] + 1) > E.TGT_MAX_SMEM


# --- each bound rejects each mutant (float64, CPU) ------------------------------------------------------------------

def _caught(got, want, bound, what):
    n = int(E.exceeds(got, want, bound).sum())
    print(f"caught: {what} ({n} values out of bound)")
    return n > 0


def _focal_case(m=E.TILE + 1, c=31, gamma=1.5):
    z, t = E.focal_rows(m, c, seed=11)
    z, t = torch.from_numpy(z), torch.from_numpy(t)
    loss, grad = R.focal_t(z, t, gamma)
    lb, gb = E.focal_bounds(z, t, gamma, grad)
    return z, t, loss, grad, lb, gb


def test_focal_bounds_reject_the_mutants():
    z, t, loss, grad, lb, gb = _focal_case()
    _, bad = R.focal_t(z, t, 1.5, mutant="pt_not_detached")
    assert _caught(bad, grad, gb, "pt not detached (gradient)")
    for gamma in (0.5, 1.5):
        z, t, loss, grad, lb, gb = _focal_case(gamma=gamma)
        bad, _ = R.focal_t(z, t, gamma, mutant="gamma_rounded")
        assert _caught(bad, loss, lb, f"gamma {gamma} rounded to an integer (loss)")
    z, t, loss, grad, lb, gb = _focal_case()
    bad, badg = R.focal_t(z, t, 1.5, mutant="tail_dropped")
    assert _caught(bad, loss, lb, "ragged tail of the last tile dropped (focal loss)")
    assert _caught(badg, grad, gb, "ragged tail of the last tile dropped (focal gradient)")
    for shape in ((3, 22, 10, 10), (1, 3, 3, 43), (2, 5, 3, 5, 7)):
        zz, tt = E.nchw_case(shape, seed=2)
        zz, tt = torch.from_numpy(zz), torch.from_numpy(tt).reshape(-1)
        rows = R.nchw_rows(zz)
        loss, grad = R.focal_t(rows, tt, 2.0)
        lb, gb = E.focal_bounds(rows, tt, 2.0, grad)
        bad, badg = R.focal_t(R.nchw_rows(zz, mutant="nhwc"), tt, 2.0)
        assert _caught(bad, loss, lb, f"{shape} read as NHWC (loss)")
        assert _caught(badg, grad, gb, f"{shape} read as NHWC (gradient)")


@pytest.mark.parametrize("n", [E.TILE + 1, 3 * E.TILE - 1])
def test_of_bounds_reject_the_mutants(n):
    pred, targ, lab = (torch.from_numpy(a) for a in E.of_case(5, n, 8, seed=4))
    loss, grad = R.of_t(pred, targ, lab)
    lb, gb = E.of_bounds(pred, targ, lab, loss, grad)
    for mutant in ("tail_dropped", "den_no_eps", "den_3x"):
        bad, badg = R.of_t(pred, targ, lab, mutant=mutant)
        caught = _caught(bad, loss, lb, f"OF n={n} {mutant} (loss)")
        if mutant == "tail_dropped":
            caught &= _caught(badg, grad, gb, f"OF n={n} {mutant} (gradient)")
        assert caught, mutant


def test_pvn3d_bounds_reject_the_mutants():
    b, n, c, k = E.PVN_B, 3 * E.TILE + 17, 22, 8
    kp, seg, ctr, kt, ct, lab = (torch.from_numpy(a) for a in E.pvn3d_case(b, n, c, k, seed=8))
    ok = torch.tensor(E.PVN_OK, dtype=torch.uint8)
    a, v = E.PVN_GRADS["both"]
    args = (kp, seg, ctr, kt, ct, lab, ok, E.PVN_WEIGHTS, E.PVN_GAMMA)
    ref = R.pvn3d_loss_t(*args, g_loss=a, g_parts=v)
    mask = ok.bool().repeat_interleave(n)
    g0 = a * E.PVN_WEIGHTS[0] + v[0]
    flb, fgb = E.focal_bounds(seg.reshape(-1, c), lab.reshape(-1), E.PVN_GAMMA, ref["d_seg"].reshape(-1, c),
                              row_mask=mask, g=g0)
    bad = R.pvn3d_loss_t(*args, g_loss=a, g_parts=v, mutant="ok_ignored")
    assert _caught(bad["parts"][0], ref["parts"][0], flb, "ok mask ignored (focal part)")
    assert _caught(bad["d_seg"].reshape(-1, c), ref["d_seg"].reshape(-1, c), fgb, "ok mask ignored (gradient)")
    assert _caught(bad["acc"], ref["acc"], 2 * E.U, "ok mask ignored (accuracy)")
    bad = R.pvn3d_loss_t(*args, g_loss=a, g_parts=v, mutant="g_parts_ignored")
    assert _caught(bad["d_seg"].reshape(-1, c), ref["d_seg"].reshape(-1, c), fgb, "g_parts ignored (d_seg)")
    _, _ = R.of_t(kp, kt, lab)
    _, kgb = E.of_bounds(kp, kt, lab, torch.zeros(b, k), ref["d_kp"])
    assert _caught(bad["d_kp"], ref["d_kp"], kgb, "g_parts ignored (d_kp)")
    # loss only, and the gradient of a term whose g is 0 (w_ctr = 0): exactly 0
    only = R.pvn3d_loss_t(*args)
    assert float(only["d_ctr"].abs().max()) == 0 and float(only["d_seg"].reshape(b, n, c)[[1, 4]].abs().max()) == 0
