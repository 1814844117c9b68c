"""TorchEval's scoring bookkeeping on the CPU, against what the reference computed (tests/golden/eval_cases.npz,
tests/golden/make_golden_eval.py): the AUC restatement, the per-class distance lists, the float64 per-slot
restatement the GPU tests use, the wrong variants the goldens must tell apart, and the refusals of
pvn3d_frame_add_adds (checked before any launch, so no device is needed)."""
import os

import numpy as np
import pytest

from pvn3d_b200 import _lib, eval_utils

import eval_ref


@pytest.fixture(scope="module")
def z(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "eval_cases.npz")))


def _ycb_meshes(z):
    off = z["ycb_mesh_off"]
    return [None] + [z["ycb_meshes"][off[c]:off[c + 1]] for c in range(1, off.size - 1)]


def _ycb_lists(z):
    cut = np.cumsum(z["ycb_list_len"])[:-1]
    return [list(x) for x in np.split(z["ycb_add_dis"], cut)], [list(x) for x in np.split(z["ycb_adds_dis"], cut)]


def _close(got, want):
    both = np.isnan(got) == np.isnan(want)
    ok = np.abs(got - want) <= 1e-5 * np.abs(want) + 1e-7
    return bool(both.all() and ok[~np.isnan(want)].all())


def test_cal_auc_equals_reference(z):
    at = 0
    for name, n, want in zip(z["auc_names"], z["auc_lens"], z["auc_values"]):
        dis = list(z["auc_dis"][at:at + n])
        at += n
        assert eval_utils.cal_auc(dis) == want, name
        assert eval_ref.cal_auc(dis) == want, name
    assert eval_utils.cal_auc([]) == 0


def test_vocap_tie_rule_is_pinned(z):
    """the precision of the FIRST element of a run of equal distances: the last one gives other numbers"""
    at, caught = 0, []
    for name, n, want in zip(z["auc_names"], z["auc_lens"], z["auc_values"]):
        dis = list(z["auc_dis"][at:at + n])
        at += n
        if eval_ref.cal_auc(dis, mutant="tie_last") != want:
            caught.append(str(name))
    assert {"ties", "many", "at_max"} <= set(caught), caught


def test_ycb_lists_and_auc_equal_reference(z):
    add_l, adds_l = [[] for _ in range(22)], [[] for _ in range(22)]
    eval_utils.append_distances(add_l, adds_l, z["ycb_add"].astype(np.float32), z["ycb_adds"].astype(np.float32),
                                z["ycb_cls_ids"])
    want_add, want_adds = _ycb_lists(z)
    assert add_l == want_add and adds_l == want_adds
    table = eval_utils.auc_table(add_l, adds_l, list(z["ycb_sym"]))
    assert table["add_auc_lst"] == list(z["ycb_add_auc"])
    assert table["adds_auc_lst"] == list(z["ycb_adds_auc"])
    assert table["add_s_auc_lst"] == list(z["ycb_add_s_auc"])
    assert table["add_auc_mean"] == np.mean(z["ycb_add_auc"][1:])


def test_scored_slots_rule(z):
    ids = z["ycb_cls_ids"]
    assert np.array_equal(eval_utils.scored_slots(ids, 22), eval_ref.slot_mask(ids, 22))
    assert np.array_equal(np.isnan(z["ycb_add"]), ~eval_ref.slot_mask(ids, 22))
    assert eval_utils.scored_slots(np.array([[3, 0, 4], [22, 1, 0]]), 22).tolist() == [[True, False, False],
                                                                                         [False, True, False]]


def test_ycb_f64_restatement_equals_reference(z):
    add, adds = eval_ref.frame_scores(z["ycb_poses"], z["ycb_present"], z["ycb_rts"], z["ycb_cls_ids"], _ycb_meshes(z),
                                      "zeros")
    assert _close(add, z["ycb_add"]) and _close(adds, z["ycb_adds"])


@pytest.mark.parametrize("mutant", ["absent_swapped", "past_zero", "cls_off_by_one", "frame_shift"])
def test_ycb_goldens_reject_mutant(z, mutant):
    add, adds = eval_ref.frame_scores(z["ycb_poses"], z["ycb_present"], z["ycb_rts"], z["ycb_cls_ids"], _ycb_meshes(z),
                                      "zeros", mutant=mutant)
    assert not (_close(add, z["ycb_add"]) and _close(adds, z["ycb_adds"]))


def test_ycb_goldens_reject_sym_swap(z):
    add_l, adds_l = _ycb_lists(z)
    sym = list(z["ycb_sym"])
    assert eval_ref.cal_auc(eval_ref.add_s_lists(add_l, adds_l, sym)[0]) == z["ycb_add_s_auc"][0]
    assert eval_ref.cal_auc(eval_ref.add_s_lists(add_l, adds_l, sym, "sym_swapped")[0]) != z["ycb_add_s_auc"][0]


@pytest.mark.parametrize("obj", [10, 4])
def test_linemod_equals_reference(z, obj):
    p = f"lm{obj}_"
    ids = np.ones((z[p + "poses"].shape[0], 1), np.int64)
    args = (z[p + "poses"], z[p + "present"], z[p + "rts"][:, :1], ids, [None, z[p + "mesh"]])
    add, adds = eval_ref.frame_scores(*args, "identity")
    assert _close(add, z[p + "add"]) and _close(adds, z[p + "adds"])
    bad_add, bad_adds = eval_ref.frame_scores(*args, "identity", mutant="absent_swapped")
    assert not (_close(bad_add, z[p + "add"]) and _close(bad_adds, z[p + "adds"]))
    add_l, adds_l = [[], []], [[], []]
    eval_utils.append_distances(add_l, adds_l, z[p + "add"].astype(np.float32), z[p + "adds"].astype(np.float32), ids)
    table = eval_utils.auc_table(add_l, adds_l, [1] if int(z[p + "sym"]) else [])
    assert table["add_auc_lst"][1] == z[p + "add_auc"] and table["adds_auc_lst"][1] == z[p + "adds_auc"]
    assert table["add_s_auc_lst"][1] == z[p + "add_s_auc"]
    assert eval_utils.lm_accuracy(add_l[1], adds_l[1], float(z[p + "diameter"])) == (z[p + "add_pct"],
                                                                                     z[p + "adds_pct"])


def test_pack_meshes_refuses_a_class_without_points():
    pts, off = eval_utils.pack_meshes({1: np.zeros((3, 3)), 2: np.ones((1, 3))})
    assert pts.shape == (4, 3) and off.tolist() == [0, 0, 3, 4]
    with pytest.raises(ValueError):
        eval_utils.pack_meshes({1: np.zeros((3, 3)), 3: np.ones((1, 3))})
    with pytest.raises(ValueError):
        eval_utils.pack_meshes({1: np.zeros((0, 3))})


def test_frame_add_adds_refusals():
    """argument checks of pvn3d_frame_add_adds, all before any launch (fake device addresses are never touched)"""
    lib = _lib.load()
    fake, ws = 4096, 8192

    def call(n_cls=3, off=(0, 0, 5, 9), b=2, slots=4, absent=0, ws_bytes=1 << 20, present=fake, add=fake):
        o = np.asarray(off, np.int32)
        return lib.pvn3d_frame_add_adds(fake, present, n_cls, fake, fake, b, slots, fake, o.ctypes.data, absent, add,
                                        fake, ws, ws_bytes, None)

    assert call(b=0) == 0 and call(slots=0) == 0                      # nothing to score: nothing launched
    assert call(n_cls=1, off=(0, 0)) == -1
    assert call(absent=2) == -1
    assert call(off=(0, 0, 5, 5)) == -1                                # class 2 has no mesh
    assert call(off=(1, 1, 5, 9)) == -1
    assert call(present=0) == -1
    n = eval_utils.ABSENT_RULES["identity"]
    assert call(absent=n, ws_bytes=16) == -4
    assert call(n_cls=65, off=tuple(range(66))) == -2
    assert call(b=300, slots=300) == -2
    assert call(off=(0, 0, 5, 0x7fffffff // 3 + 1)) == -2
    assert lib.pvn3d_frame_add_adds_workspace_bytes(2, 4, 2049) == 8 * 9 * 8 + 256
    assert lib.pvn3d_frame_add_adds_workspace_bytes(300, 300, 10) == 0
