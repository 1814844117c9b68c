"""Record TorchEval's scoring from the REFERENCE ITSELF on the CPU (run in the build container only).

    python tests/golden/make_golden_eval.py

Imports the unmodified reference Python from the checkout at REF (with the import shims of pvn3d_b200.compat and
the `.cuda()` no-op of make_golden_cpu.py) and records, into eval_cases.npz:
  ycb_*   four synthetic frames through `eval_metric` (pvn3d_eval_utils.py:113-137), merged in frame order as
          eval_pose_parallel does (:380-387): predicted, absent (zero pose) and relabel-lost (identity) classes, a
          false positive, a repeated class, a 0 in the middle of cls_ids, symmetric classes, distances past 0.1 m;
          then TorchEval.cal_auc (:249-296): its pickle and its printed lines.
  lm<obj>_* five frames through `eval_metric_lm` (:204-220) for a symmetric and a plain LineMOD object, one of them
          with an empty mask (identity pose); then TorchEval.cal_lm_add (:298-343).
  auc_*   Basic_Utils.cal_auc (basic_utils.py:597-604) edge cases: empty, one value, all > 0.1, values of exactly
          0.1, runs of tied distances.
Meshes are a few hundred points, so the reference's [P,P,3] stays cheap.  `config.log_eval_dir` goes to a temporary
directory.  While recording, the float64 restatement of tests/eval_ref.py is checked against every reference value
(1e-5 relative + 1e-7 m) and pvn3d_b200.eval_utils' AUC and list bookkeeping bit for bit; a mismatch aborts.
"""
import contextlib
import glob
import io
import os
import pickle
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
REF = "/root/reference/pvn3d"
OUT = os.path.dirname(os.path.abspath(__file__))

from pvn3d_b200 import compat, synth  # noqa: E402
from pvn3d_b200 import eval_utils as ours  # noqa: E402
from oracle import ext_cpu  # noqa: E402
import eval_ref  # noqa: E402

compat.install_import_shims()
sys.modules["lib.pointnet2_utils._ext"] = ext_cpu
sys.path.insert(0, REF)
torch.Tensor.cuda = lambda self, *a, **k: self          # run the reference's .cuda() code on CPU
torch.nn.Module.cuda = lambda self, *a, **k: self

from lib.utils import pvn3d_eval_utils as ref_eval      # noqa: E402

N_CLS = 22
LM_OBJS = (10, 4)    # eggbox (symmetric), cam


def _pose(rng, t_scale=1.0):
    R = synth._haar_rotation(rng)
    t = rng.uniform([-0.2, -0.2, 0.6], [0.2, 0.2, 1.0]) * t_scale
    return np.concatenate([R, t[:, None]], 1).astype(np.float32)


def _perturb(rng, rt, ang, off):
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    dR = np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K
    out = np.concatenate([dR @ rt[:, :3].astype(np.float64), (rt[:, 3] + rng.normal(0, off, 3))[:, None]], 1)
    return out.astype(np.float32)


def _mesh(rng, n, sym):
    m = rng.uniform(-0.06, 0.06, size=(n, 3)) * rng.uniform(0.5, 1.5, 3)
    if sym:
        m = np.concatenate([m[: n // 2], -m[: n - n // 2]], 0)
    return m.astype(np.float32)


def _close(a, b):
    return abs(a - b) <= 1e-5 * abs(b) + 1e-7


@contextlib.contextmanager
def _eval_dir():
    with tempfile.TemporaryDirectory() as d:
        prev = ref_eval.config.log_eval_dir, ref_eval.config_lm.log_eval_dir
        ref_eval.config.log_eval_dir = ref_eval.config_lm.log_eval_dir = d
        try:
            yield d
        finally:
            ref_eval.config.log_eval_dir, ref_eval.config_lm.log_eval_dir = prev


def _run_and_capture(fn):
    with _eval_dir() as d:
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            fn()
        (pkl,) = glob.glob(os.path.join(d, "*.pkl"))
        with open(pkl, "rb") as f:
            return buf.getvalue(), os.path.basename(pkl), pickle.load(f)


def _slot_values(per_frame_lists, ids, scored):
    """[B,I] values of the scored slots, read back from each frame's class-0 list (slot order), NaN elsewhere"""
    out = np.full(ids.shape, np.nan)
    for f, lst in enumerate(per_frame_lists):
        js = np.nonzero(scored[f])[0]
        assert len(js) == len(lst[0]), (f, len(js), len(lst[0]))
        out[f, js] = lst[0]
    return out


def golden_ycb(out):
    rng = np.random.default_rng(2026)
    sym = ref_eval.config.ycb_sym_cls_ids
    meshes = [None] + [_mesh(rng, int(rng.integers(40, 320)), c in sym) for c in range(1, N_CLS)]
    meshes[5] = meshes[5][:1]                                       # a one-point mesh
    bs = ref_eval.bs_utils
    for c in range(1, N_CLS):
        bs.ycb_cls_ptsxyz_cuda_dict[ref_eval.cls_lst[c - 1]] = torch.from_numpy(meshes[c])
    slots = [[3, 7, 13, 16],                 # all predicted; 13, 16 symmetric
             [5, 16, 2, 21, 11],             # 16 and 21 not predicted (zero pose); a one-point mesh
             [1, 4, 0, 9, 11],               # a 0 in the middle: 9 and 11 are not scored
             [21, 20, 19, 8, 6, 6]]          # 8 predicted but lost in the relabel pass (identity); 6 twice
    predicted = [[3, 7, 13, 16, 18], [5, 2, 11], [1, 4, 9, 11], [21, 20, 19, 8, 6, 12]]
    B = len(slots)
    poses = np.zeros((B, N_CLS, 3, 4), np.float32)
    present = np.zeros((B, N_CLS), np.uint8)
    rts = np.zeros((B, N_CLS, 3, 4), np.float32)
    ids = np.zeros((B, N_CLS), np.int64)
    for f in range(B):
        for i, c in enumerate(slots[f]):
            ids[f, i] = c
            rts[f, i] = _pose(rng)
        for c in predicted[f]:
            present[f, c] = 1
            hit = [i for i, x in enumerate(slots[f]) if x == c]
            base = rts[f, hit[0]] if hit else _pose(rng)
            k = int(rng.integers(0, 4))
            poses[f, c] = _perturb(rng, base, [0.0, 0.02, 0.1, 0.6][k], [0.0, 0.003, 0.02, 0.15][k])
    poses[3, 8] = np.eye(4, dtype=np.float32)[:3]                  # relabel-lost: cal_frame_poses appends identity
    poses[2, 9] = poses[2, 11] = 0.0                                # not scored anyway (after the 0)
    merged_add = [[] for _ in range(N_CLS)]
    merged_adds = [[] for _ in range(N_CLS)]
    frames_add, frames_adds = [], []
    for f in range(B):
        pred_cls_ids = np.nonzero(present[f])[0]
        pred_pose_lst = [poses[f, c].astype(np.float64) for c in pred_cls_ids]
        a, s = ref_eval.eval_metric(torch.from_numpy(ids[f][:, None]), pred_pose_lst, pred_cls_ids,
                                    torch.from_numpy(rts[f]), None, None)
        frames_add.append(a)
        frames_adds.append(s)
        for i in range(N_CLS):
            merged_add[i] += a[i]
            merged_adds[i] += s[i]
    scored = eval_ref.slot_mask(ids, N_CLS)
    add = _slot_values(frames_add, ids, scored)
    adds = _slot_values(frames_adds, ids, scored)
    # checks of the restatements against what the reference computed
    ra, rs = eval_ref.frame_scores(poses, present, rts, ids, meshes, "zeros")
    for f, i in zip(*np.nonzero(scored)):
        assert _close(ra[f, i], add[f, i]) and _close(rs[f, i], adds[f, i]), (f, i, ra[f, i], add[f, i])
    mine_add, mine_adds = [[] for _ in range(N_CLS)], [[] for _ in range(N_CLS)]
    ours.append_distances(mine_add, mine_adds, add.astype(np.float32), adds.astype(np.float32), ids)
    assert mine_add == merged_add and mine_adds == merged_adds
    te = ref_eval.TorchEval()
    te.cls_add_dis = [list(x) for x in merged_add]
    te.cls_adds_dis = [list(x) for x in merged_adds]
    text, name, sv = _run_and_capture(te.cal_auc)
    table = ours.auc_table(merged_add, merged_adds, sym)
    for k in ("add_auc_lst", "adds_auc_lst", "add_s_auc_lst"):
        assert table[k] == sv[k], (k, table[k], sv[k])
    print(text)
    lens = np.array([len(x) for x in merged_add], np.int32)
    out.update(ycb_meshes=np.concatenate(meshes[1:], 0),
               ycb_mesh_off=np.concatenate([[0, 0], np.cumsum([len(m) for m in meshes[1:]])]).astype(np.int32),
               ycb_poses=poses, ycb_present=present, ycb_rts=rts, ycb_cls_ids=ids.astype(np.int32),
               ycb_add=add, ycb_adds=adds, ycb_sym=np.array(sym, np.int32),
               ycb_list_len=lens, ycb_add_dis=np.concatenate(merged_add), ycb_adds_dis=np.concatenate(merged_adds),
               ycb_add_auc=np.array(sv["add_auc_lst"]), ycb_adds_auc=np.array(sv["adds_auc_lst"]),
               ycb_add_s_auc=np.array(sv["add_s_auc_lst"]), ycb_pkl_name=np.array(name), ycb_printed=np.array(text))


def golden_lm(out, obj_id):
    rng = np.random.default_rng(100 + obj_id)
    cfg = ref_eval.config_lm
    mesh = _mesh(rng, 300, obj_id in cfg.lm_sym_cls_ids)
    ref_eval.bs_utils_lm.lm_cls_ptsxyz_cuda_dict[obj_id] = torch.from_numpy(mesh)
    B = 5
    poses = np.zeros((B, 2, 3, 4), np.float32)
    present = np.zeros((B, 2), np.uint8)
    rts = np.zeros((B, 2, 3, 4), np.float32)          # eval_metric_lm reads RTs[0] only
    merged_add = [[] for _ in range(N_CLS)]
    merged_adds = [[] for _ in range(N_CLS)]
    for f in range(B):
        rts[f, 0] = _pose(rng)
        if f == 2:                                       # empty mask: cal_frame_poses_lm appends the identity
            poses[f, 1] = np.eye(4, dtype=np.float32)[:3]
        else:
            present[f, 1] = 1
            poses[f, 1] = _perturb(rng, rts[f, 0], [0.0, 0.05, 0.3, 0.01, 0.02][f], [0.0, 0.005, 0.05, 0.001, 0.0][f])
        a, s = ref_eval.eval_metric_lm(None, [poses[f, 1].astype(np.float64)], torch.from_numpy(rts[f]), None, None,
                                       obj_id)
        for i in range(N_CLS):
            merged_add[i] += a[i]
            merged_adds[i] += s[i]
    ids = np.ones((B, 1), np.int64)
    add = np.array(merged_add[obj_id])[:, None]
    adds = np.array(merged_adds[obj_id])[:, None]
    ra, rs = eval_ref.frame_scores(poses, present, rts[:, :1], ids, [None, mesh], "identity")
    for f in range(B):
        assert _close(ra[f, 0], add[f, 0]) and _close(rs[f, 0], adds[f, 0]), (f, ra[f, 0], add[f, 0])
    te = ref_eval.TorchEval()
    te.cls_add_dis = [list(x) for x in merged_add]
    te.cls_adds_dis = [list(x) for x in merged_adds]
    text, name, sv = _run_and_capture(lambda: te.cal_lm_add(obj_id))
    diameter = cfg.lm_r_lst[obj_id]["diameter"] / 1000.0
    sym = [1] if obj_id in cfg.lm_sym_cls_ids else []
    table = ours.auc_table([merged_add[0], merged_add[obj_id]], [merged_adds[0], merged_adds[obj_id]], sym)
    assert [table[k][1] for k in ("add_auc_lst", "adds_auc_lst", "add_s_auc_lst")] == \
        [sv[k][0] for k in ("add_auc_lst", "adds_auc_lst", "add_s_auc_lst")]
    assert ours.lm_accuracy(merged_add[obj_id], merged_adds[obj_id], diameter) == (sv["add"], sv["adds"])
    print(text)
    p = f"lm{obj_id}_"
    out.update({p + "mesh": mesh, p + "poses": poses, p + "present": present, p + "rts": rts, p + "add": add,
                p + "adds": adds, p + "diameter": np.float64(diameter), p + "sym": np.int32(len(sym)),
                p + "add_auc": np.float64(sv["add_auc_lst"][0]), p + "adds_auc": np.float64(sv["adds_auc_lst"][0]),
                p + "add_s_auc": np.float64(sv["add_s_auc_lst"][0]), p + "add_pct": np.float64(sv["add"]),
                p + "adds_pct": np.float64(sv["adds"]), p + "pkl_name": np.array(name), p + "printed": np.array(text)})


def golden_auc(out):
    rng = np.random.default_rng(5)
    cases = {
        "empty": [],
        "one": [0.042],
        "one_far": [0.3],
        "all_far": list(rng.uniform(0.11, 0.5, 7)),
        "at_max": [0.1, 0.1, 0.05, 0.1],
        "ties": [0.02, 0.05, 0.02, 0.07, 0.05, 0.05, 0.01, 0.2, 0.07, 0.02],
        "many": list(np.round(rng.uniform(0.0, 0.12, 400), 3)),   # rounded: long runs of equal distances
    }
    names = sorted(cases)
    vals = []
    for k in names:
        v = ref_eval.bs_utils.cal_auc(cases[k])
        assert ours.cal_auc(cases[k]) == v, (k, ours.cal_auc(cases[k]), v)
        vals.append(v)
        print(f"  cal_auc {k}: {v!r}")
    out.update(auc_names=np.array(names), auc_values=np.array(vals, np.float64),
               auc_lens=np.array([len(cases[k]) for k in names], np.int32),
               auc_dis=np.concatenate([np.asarray(cases[k], np.float64) for k in names]))


if __name__ == "__main__":
    out = {}
    golden_ycb(out)
    for obj in LM_OBJS:
        golden_lm(out, obj)
    golden_auc(out)
    out["lm_objs"] = np.array(LM_OBJS, np.int32)
    np.savez_compressed(os.path.join(OUT, "eval_cases.npz"), **out)
    print("done:", os.path.getsize(os.path.join(OUT, "eval_cases.npz")), "bytes")
