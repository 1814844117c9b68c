"""The float64 restatements of tests/train_ref.py against the goldens recorded from the reference's get_item and
lib/loss.py (tests/golden/train_cases.npz, tests/golden/make_golden_train.py), the mutants those goldens must reject,
and the argument refusals of the training entry points, which happen before any launch (no GPU needed)."""
import ctypes
import os

import numpy as np
import pytest
import torch

import train_ref as R
from pvn3d_b200 import _lib


@pytest.fixture(scope="module")
def gold(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "train_cases.npz")))


def _targets(g, mutant=None):
    return R.targets_ref(g["tgt_pcld"], g["tgt_labels"], g["tgt_slot_ids"], g["tgt_rts64"], g["tgt_kp_table"],
                         g["tgt_ctr_table"], mutant=mutant)


def test_targets_ref_reproduces_get_item(gold):
    kp, ctr, kp3, ctr3 = _targets(gold)
    assert R.digest(kp) == str(gold["tgt_kp_targ_ofst_sha256"])          # every element, bit for bit
    assert np.array_equal(kp[:, ::R.ROW_STRIDE], gold["tgt_kp_targ_ofst_rows"])
    for got, name in ((ctr, "ctr_targ_ofst"), (kp3, "kp3ds"), (ctr3, "ctr3ds")):
        assert np.array_equal(got, gold["tgt_" + name]), name
    # cld_rgb_nrm is the sampled cloud, its colours and get_normal's (stubbed) zeros
    cld = R.cld_rgb_nrm_of(gold["tgt_pcld"], gold["tgt_rgb"], gold["tgt_choose"])
    assert R.digest(cld) == str(gold["tgt_cld_rgb_nrm_sha256"])
    # get_item's own slot outputs agree with the recorded meta slots
    assert np.array_equal(gold["tgt_cls_ids"][..., 0], gold["tgt_slot_ids"])
    assert np.array_equal(gold["tgt_RTs"], gold["tgt_rts64"].astype(np.float32))


def test_golden_frames_cover_the_cases(gold):
    ids, lab = gold["tgt_slot_ids"], gold["tgt_labels"]
    assert any(len(set(r[r > 0])) < (r > 0).sum() for r in ids), "no class listed twice in meta"
    assert any(not set(np.unique(l[l > 0])) <= set(r) for l, r in zip(lab, ids)), "no label without a meta entry"
    choose = gold["tgt_choose"][:, 0]
    assert any(len(np.unique(c)) < c.size for c in choose), "no frame padded by 'wrap'"


def test_first_slot_wins_is_rejected(gold):
    bad = _targets(gold, "first_slot_wins")
    assert R.digest(bad[0]) != str(gold["tgt_kp_targ_ofst_sha256"])
    assert not np.array_equal(bad[1], gold["tgt_ctr_targ_ofst"])


def test_focal_ref_reproduces_lib_loss(gold):
    detached_told_apart = False
    for i in range(int(gold["n_focal"])):
        z, t, gamma = gold[f"focal{i}_z"], gold[f"focal{i}_t"], float(gold[f"focal{i}_gamma"])
        loss, grad = R.focal_ref(z, t, gamma)
        want = float(gold[f"focal{i}_loss"])
        assert abs(loss - want) <= 1e-12 * abs(want), i
        np.testing.assert_allclose(grad, gold[f"focal{i}_grad"], rtol=1e-12, atol=1e-300)
        _, bad = R.focal_ref(z, t, gamma, mutant="pt_not_detached")
        detached_told_apart |= not np.allclose(bad, gold[f"focal{i}_grad"], rtol=1e-6, atol=1e-12)
    assert detached_told_apart


def test_of_ref_reproduces_lib_loss(gold):
    for i in range(int(gold["n_of"])):
        args = gold[f"of{i}_pred"], gold[f"of{i}_targ"], gold[f"of{i}_labels"], gold[f"of{i}_g"]
        loss, grad = R.of_ref(*args)
        np.testing.assert_allclose(loss, gold[f"of{i}_loss"], rtol=1e-12, atol=0)
        np.testing.assert_allclose(grad, gold[f"of{i}_grad"], rtol=1e-12, atol=0)
        bad, _ = R.of_ref(*args, mutant="den_3x")
        assert not np.allclose(bad, gold[f"of{i}_loss"], rtol=1e-3)   # the loss is 3x smaller
    # a frame without labelled points: loss and gradient 0
    lab = gold["of1_labels"]
    assert (lab[1] == 0).all() and (gold["of1_loss"][1] == 0).all() and (gold["of1_grad"][1] == 0).all()


# --- refusals before any launch: the C entry points validate on the host, the pointers are never read -------------

_FAKE = 1 << 20


def test_train_targets_refusals():
    lib = _lib.load()
    P = _FAKE
    ok_args = [P] * 4 + [2, 100, 22, P, P, 22, 8, P, P, P, P, 0]
    for i in range(4):
        a = list(ok_args)
        a[i] = 0
        assert lib.pvn3d_train_targets(*a) == -1
    for idx, bad, rc in ((4, 0, -1), (5, 0, -1), (6, 0, -1), (9, 0, -1), (10, 0, -1),
                         (4, 70000, -2), (9, 5000, -2), (6, 2000, -2), (10, 400, -2)):
        a = list(ok_args)
        a[idx] = bad
        assert lib.pvn3d_train_targets(*a) == rc, (idx, bad)


def _loss_args(**kw):
    a = _lib.LossArgs()
    a.seg, a.seg_target, a.seg_rows, a.n_cls, a.seg_inner, a.gamma, a.seg_mean = _FAKE, _FAKE, 24 * 12288, 22, 1, 2.0, 1
    a.kp_pred, a.kp_targ, a.n_kp = _FAKE, _FAKE, 8
    a.ctr_pred, a.ctr_targ, a.n_ctr = _FAKE, _FAKE, 1
    a.labels, a.b, a.n, a.ok = _FAKE, 24, 12288, 0
    a.w_seg, a.w_kp, a.w_ctr = 2.0, 1.0, 1.0
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("bad", [dict(seg=0, kp_pred=0, ctr_pred=0), dict(seg_target=0), dict(seg_rows=0),
                                 dict(n_cls=0), dict(gamma=-1.0), dict(gamma=float("nan")), dict(gamma=float("inf")),
                                 dict(seg_inner=5), dict(labels=0), dict(kp_targ=0), dict(n_kp=0), dict(b=0),
                                 dict(ok=_FAKE, seg_rows=1000)])
def test_train_loss_invalid_arguments(bad):
    lib = _lib.load()
    a = _loss_args(**bad)
    assert lib.pvn3d_train_loss_workspace_bytes(ctypes.byref(a)) == 0
    assert lib.pvn3d_train_loss_forward(ctypes.byref(a), 0, 0, 0, 0, 0, _FAKE * 256, 1 << 30, 0) == -1


@pytest.mark.parametrize("bad", [dict(n_cls=129), dict(n_kp=49), dict(n_ctr=49)])
def test_train_loss_unsupported_sizes(bad):
    lib = _lib.load()
    a = _loss_args(**bad)
    assert lib.pvn3d_train_loss_workspace_bytes(ctypes.byref(a)) == 0
    assert lib.pvn3d_train_loss_forward(ctypes.byref(a), 0, 0, 0, 0, 0, _FAKE * 256, 1 << 30, 0) == -2


def test_train_loss_workspace_refusals():
    lib = _lib.load()
    a = _loss_args()
    need = lib.pvn3d_train_loss_workspace_bytes(ctypes.byref(a))
    assert need > 0
    assert lib.pvn3d_train_loss_forward(ctypes.byref(a), 0, 0, 0, 0, 0, _FAKE * 256, need - 1, 0) == -4
    assert lib.pvn3d_train_loss_forward(ctypes.byref(a), 0, 0, 0, 0, 0, _FAKE * 256 + 4, need, 0) == -1
    assert lib.pvn3d_train_loss_backward(ctypes.byref(a), 0, 0, 0, _FAKE, _FAKE, _FAKE, _FAKE * 256, need, 0) == -1


def test_python_refusals_without_a_device():
    from pvn3d_b200 import train_utils as T

    with pytest.raises(ValueError):
        T.FocalLoss(gamma=2, alpha=0.25)
    with pytest.raises(ValueError):
        T.FocalLoss(gamma=-1)
    with pytest.raises(ValueError):
        T.PVN3DLoss(weights=(1, 1))
    with pytest.raises(RuntimeError, match="CUDA"):
        T.FocalLoss(gamma=2)(torch.zeros(4, 3), torch.zeros(4, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="CUDA"):
        T.OFLoss()(torch.zeros(1, 8, 4, 3), torch.zeros(1, 4, 8, 3), torch.zeros(1, 4, dtype=torch.int64))
    with pytest.raises(ValueError):
        T.TrainTargets(kp_table=np.zeros((22, 8, 3)), ctr_table=np.zeros((21, 3)), device="cuda:0")
    with pytest.raises(RuntimeError):
        T.TrainTargets(device="cpu")
