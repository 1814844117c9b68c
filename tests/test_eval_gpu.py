"""pvn3d_frame_add_adds, PoseEvaluator and the batched TorchEval.eval_pose_parallel on the GPU: against the float64
brute force of tests/eval_ref.py, against pvn3d_pose_add_adds bit for bit, under CUDA graph capture, against the
reference's recorded scoring (tests/golden/eval_cases.npz) and, where the reference Python is staged
(oracle/_ref/py), against the reference's own eval_pose_parallel; plus the per-frame cal_frame_poses under two
interleaved threads."""
import glob
import os
import pickle
import threading

import numpy as np
import pytest
import torch

from pvn3d_b200 import compat, eval_utils, synth
from pvn3d_b200.eval_utils import FramePoseSolver, PoseEvaluator

import eval_ref
from helpers import load_reference_python

pytestmark = pytest.mark.gpu


def _close(got, want, what=""):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)), what
    m = ~np.isnan(want)
    err = np.abs(got[m] - want[m]) - (1e-5 * np.abs(want[m]) + 1e-7)
    assert err.size == 0 or err.max() <= 0, (what, float(err.max()))


def _rt(rng, n):
    out = np.zeros((n, 3, 4), np.float32)
    for k in range(n):
        out[k, :, :3] = synth._haar_rotation(rng)
        out[k, :, 3] = rng.uniform([-0.2, -0.2, 0.5], [0.2, 0.2, 1.0])
    return out


def _case(rng, b, slots, sizes, absent_frac=0.3):
    n_cls = len(sizes) + 1
    meshes = [None] + [rng.uniform(-0.08, 0.08, (p, 3)).astype(np.float32) for p in sizes]
    gt = _rt(rng, b * slots).reshape(b, slots, 3, 4)
    ids = rng.integers(1, n_cls, (b, slots)).astype(np.int32)
    if slots > 3:
        ids[0, slots // 2] = 0                                   # a 0 in the middle of frame 0
        ids[-1, slots - 2:] = 0                                  # zero padding at the end
    poses = (gt.reshape(b * slots, 12)[rng.integers(0, b * slots, b * n_cls)].reshape(b, n_cls, 3, 4) +
             rng.normal(0, 0.01, (b, n_cls, 3, 4))).astype(np.float32)
    for f in range(b):                                           # predictions near the ground truth of each slot
        for i in range(slots):
            poses[f, ids[f, i]] = gt[f, i] + rng.normal(0, 0.005, (3, 4)).astype(np.float32)
    present = (rng.uniform(size=(b, n_cls)) > absent_frac).astype(np.uint8)
    return meshes, poses, present, gt, ids


@pytest.mark.parametrize("absent", ["zeros", "identity"])
@pytest.mark.parametrize("b,slots,sizes", [
    (1, 22, [1, 2047, 2048, 2049, 300]),                        # B = 1, I = 22, tile edges, P = 1
    (3, 5, [4100, 17, 2000, 1, 2049, 256, 257]),                 # ragged meshes across tiles
    (16, 5, [2000] * 21),                                        # YCB-shape batch
])
def test_frame_add_adds_against_float64(cuda_dev, absent, b, slots, sizes):
    rng = np.random.default_rng(b * 100 + slots + len(sizes))
    meshes, poses, present, gt, ids = _case(rng, b, slots, sizes)
    want_add, want_adds = eval_ref.frame_scores(poses, present, gt, ids, meshes, absent)
    ev = PoseEvaluator({c: m for c, m in enumerate(meshes) if c}, absent=absent, device=cuda_dev)
    big = torch.zeros((b + 4,) + poses.shape[1:], device=cuda_dev)          # a solver sized for a larger batch
    big[:b] = torch.from_numpy(poses).to(cuda_dev)
    pres = torch.zeros((b + 4, poses.shape[1]), dtype=torch.uint8, device=cuda_dev)
    pres[:b] = torch.from_numpy(present).to(cuda_dev)
    add, adds = ev.add_batch(big[:b], pres[:b], torch.from_numpy(gt).to(cuda_dev), torch.from_numpy(ids).to(cuda_dev))
    _close(add.cpu().numpy(), want_add, "add")
    _close(adds.cpu().numpy(), want_adds, "adds")
    lists_add, lists_adds = ev.distances()
    assert len(lists_add[0]) == int(eval_ref.slot_mask(ids, len(meshes)).sum())


def test_pose_add_adds_is_the_one_mesh_frame_call(cuda_dev):
    rng = np.random.default_rng(4)
    for p in (1, 2047, 2048, 2049, 7001):
        mesh = torch.from_numpy(rng.uniform(-0.1, 0.1, (p, 3)).astype(np.float32)).to(cuda_dev)
        gt = torch.from_numpy(_rt(rng, 9)).to(cuda_dev)
        pr = gt + torch.from_numpy(rng.normal(0, 0.02, (9, 3, 4)).astype(np.float32)).to(cuda_dev)
        a1, s1 = eval_utils.pose_add_adds(pr, gt, mesh)
        poses = torch.zeros((9, 2, 3, 4), device=cuda_dev)
        poses[:, 1] = pr
        present = torch.ones((9, 2), dtype=torch.uint8, device=cuda_dev)
        ids = torch.ones((9, 1), dtype=torch.int32, device=cuda_dev)
        _, off = eval_utils.pack_meshes({1: mesh})
        a2, s2 = eval_utils.frame_add_adds(poses, present, gt[:, None], ids, mesh, off)
        assert torch.equal(a1, a2[:, 0]) and torch.equal(s1, s2[:, 0]), p


def test_add_batch_under_graph_capture(cuda_dev):
    rng = np.random.default_rng(8)
    meshes, poses, present, gt, ids = _case(rng, 4, 6, [500, 2049, 3, 1200])
    ev = PoseEvaluator({c: m for c, m in enumerate(meshes) if c}, sym_cls_ids=[2], device=cuda_dev)
    args = [torch.from_numpy(x).to(cuda_dev) for x in (poses, present, gt, ids)]
    want = [t.clone() for t in ev.add_batch(*args)]
    ev.reset()
    s = torch.cuda.Stream(cuda_dev)
    s.wait_stream(torch.cuda.current_stream(cuda_dev))
    with torch.cuda.stream(s):
        ev.add_batch(*args)                                      # warm-up outside the capture
    torch.cuda.current_stream(cuda_dev).wait_stream(s)
    ev.reset()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        add, adds = ev.add_batch(*args)
    g.replay()
    torch.cuda.synchronize(cuda_dev)
    assert torch.equal(add.view(torch.int32), want[0].view(torch.int32))       # same bits, the NaNs included
    assert torch.equal(adds.view(torch.int32), want[1].view(torch.int32))


def test_evaluator_on_reference_goldens(cuda_dev, golden_dir):
    z = dict(np.load(os.path.join(golden_dir, "eval_cases.npz")))
    off = z["ycb_mesh_off"]
    meshes = {c: z["ycb_meshes"][off[c]:off[c + 1]] for c in range(1, off.size - 1)}
    ev = PoseEvaluator(meshes, list(z["ycb_sym"]), device=cuda_dev)
    t = [torch.from_numpy(z[k]).to(cuda_dev) for k in ("ycb_poses", "ycb_present", "ycb_rts", "ycb_cls_ids")]
    ev.add_batch(t[0][:2], t[1][:2], t[2][:2], t[3][:2, :, None])          # two batches: the order spans them
    ev.add_batch(t[0][2:], t[1][2:], t[2][2:], t[3][2:, :, None])
    add, adds = ev.distances()
    cut = np.cumsum(z["ycb_list_len"])[:-1]
    for got, want in ((add, np.split(z["ycb_add_dis"], cut)), (adds, np.split(z["ycb_adds_dis"], cut))):
        assert [len(x) for x in got] == [len(x) for x in want]
        for g, w in zip(got, want):
            _close(g, w)
    res = ev.auc()
    for k, key in (("add_auc_lst", "ycb_add_auc"), ("adds_auc_lst", "ycb_adds_auc"), ("add_s_auc_lst", "ycb_add_s_auc")):
        assert np.abs(np.asarray(res[k], np.float64) - z[key]).max() <= 1e-6, k
    for obj in z["lm_objs"]:
        p = f"lm{int(obj)}_"
        ev = PoseEvaluator({1: z[p + "mesh"]}, [1] if int(z[p + "sym"]) else [], {1: float(z[p + "diameter"])},
                           absent="identity", device=cuda_dev)
        n = z[p + "poses"].shape[0]
        ev.add_batch(torch.from_numpy(z[p + "poses"]).to(cuda_dev), torch.from_numpy(z[p + "present"]).to(cuda_dev),
                     torch.from_numpy(z[p + "rts"][:, :1]).to(cuda_dev), torch.ones((n, 1), dtype=torch.int32, device=cuda_dev))
        add, adds = ev.distances()
        _close(add[1], z[p + "add"][:, 0])
        _close(adds[1], z[p + "adds"][:, 0])
        res = ev.auc()
        assert abs(res["add_auc_lst"][1] - z[p + "add_auc"]) <= 1e-6
        assert abs(res["add_s_auc_lst"][1] - z[p + "add_s_auc"]) <= 1e-6
        assert ev.lm_accuracy(1) == (z[p + "add_pct"], z[p + "adds_pct"])


def test_per_frame_cal_frame_poses_interleaved(cuda_dev, monkeypatch):
    """two threads call cal_frame_poses on different frames; both solves are enqueued before either host copy
    whenever nothing serialises them.  Each call must get its own frame's poses."""
    frames = [synth.make_frame("ycb", n_points=4096, seed=s) for s in (61, 62)]
    args = [[torch.from_numpy(x).to(cuda_dev) for x in (f.pcld, f.labels, f.ctr_of, f.kp_of)] for f in frames]
    alone = [eval_utils.cal_frame_poses(*a, True, 22, True) for a in args]
    torch.cuda.synchronize(cuda_dev)
    barrier = threading.Barrier(2)
    orig = FramePoseSolver.solve

    def solve(self, *a):
        out = orig(self, *a)
        try:
            barrier.wait(timeout=3.0)          # wait for the other thread's solve (a lock makes this time out)
        except threading.BrokenBarrierError:
            pass
        return out

    monkeypatch.setattr(FramePoseSolver, "solve", solve)
    got = [None, None]

    def run(k):
        got[k] = eval_utils.cal_frame_poses(*args[k], True, 22, True)

    threads = [threading.Thread(target=run, args=(k,)) for k in (0, 1)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=60)
    assert not any(t.is_alive() for t in threads)
    for k in (0, 1):
        assert np.array_equal(got[k][0], alone[k][0])
        assert all(np.array_equal(p, q) for p, q in zip(got[k][1], alone[k][1])), k


def _batch_inputs(shape, b, n, dev, obj_id=None):
    frames = [synth.make_frame(shape, n_points=n, seed=300 + i, lm_obj_id=obj_id) for i in range(b)]
    n_obj = 22
    rts = np.zeros((b, n_obj, 3, 4), np.float32)
    ids = np.zeros((b, n_obj, 1), np.int64)
    for f, fr in enumerate(frames):
        k = len(fr.cls_ids)
        rts[f, :k] = fr.RTs
        ids[f, :k, 0] = fr.cls_ids
    if shape == "ycb":
        ids[1, 1, 0] = 0                               # a 0 in the middle
        lab = [fr.labels.copy() for fr in frames]
        lab[2][lab[2] == frames[2].cls_ids[0]] = 0     # a ground-truth object the frame does not predict
    else:
        lab = [fr.labels.copy() for fr in frames]
        lab[1][:] = 0                                  # an empty mask
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
    return dict(pclds=t(np.stack([fr.pcld for fr in frames])), masks=t(np.stack(lab)).long(),
                pred_ctr_ofs=t(np.stack([fr.ctr_of for fr in frames])), cls_ids=t(ids), RTs=t(rts),
                pred_kp_ofs=t(np.stack([fr.kp_of for fr in frames])))


@pytest.mark.parametrize("shape", ["ycb", "linemod"])
def test_dropin_eval_pose_parallel_vs_reference(cuda_dev, shape, tmp_path):
    ref = load_reference_python()
    if ref is None:
        pytest.skip("reference Python not staged under oracle/_ref/py")
    ev_mod = ref.eval_utils
    rng = np.random.default_rng(9)
    obj_id = 10 if shape == "linemod" else 0
    if shape == "ycb":
        for c in range(1, 22):
            ev_mod.bs_utils.ycb_cls_ptsxyz_cuda_dict[ev_mod.cls_lst[c - 1]] = torch.from_numpy(
                rng.uniform(-0.06, 0.06, (int(rng.integers(200, 700)), 3)).astype(np.float32)).to(cuda_dev)
    else:
        ev_mod.bs_utils_lm.lm_cls_ptsxyz_cuda_dict[obj_id] = torch.from_numpy(
            rng.uniform(-0.06, 0.06, (2000, 3)).astype(np.float32)).to(cuda_dev)
    inp = _batch_inputs(shape, 4, 4096, cuda_dev, obj_id=obj_id if shape == "linemod" else None)
    kw = dict(use_ctr_clus_flter=shape == "ycb", use_ctr=True, min_cnt=1, use_p2d=False)
    if shape == "linemod":
        kw.update(ds_type="linemod", obj_id=obj_id)
    cls = ev_mod.TorchEval
    orig = cls.eval_pose_parallel
    saved = (ev_mod.cal_frame_poses, ev_mod.cal_frame_poses_lm, ev_mod.MeanShiftTorch, ref.meanshift.MeanShiftTorch)
    compat.patch_post_modules()                        # both sides solve the poses with this package's solver
    teams = []
    try:
        for patched in (False, True):
            if patched:
                compat.patch_eval_pose_parallel(cls)
            te = cls()
            for rep in range(2):                       # two calls: the lists keep growing in order
                te.eval_pose_parallel(inp["pclds"], None, inp["masks"], inp["pred_ctr_ofs"], None, inp["masks"], rep,
                                      inp["cls_ids"], inp["RTs"], inp["pred_kp_ofs"], **kw)
            teams.append(te)
    finally:
        cls.eval_pose_parallel = orig
        ev_mod.cal_frame_poses, ev_mod.cal_frame_poses_lm, ev_mod.MeanShiftTorch, ref.meanshift.MeanShiftTorch = saved
    want, got = teams
    assert sum(len(x) for x in got.cls_add_dis) > 0
    for a, b in ((got.cls_add_dis, want.cls_add_dis), (got.cls_adds_dis, want.cls_adds_dis)):
        assert [len(x) for x in a] == [len(x) for x in b]
        for x, y in zip(a, b):
            _close(x, y)
    pk = []
    for k, te in enumerate(teams):
        d = tmp_path / str(k)
        d.mkdir()
        prev = ev_mod.config.log_eval_dir, ev_mod.config_lm.log_eval_dir
        ev_mod.config.log_eval_dir = ev_mod.config_lm.log_eval_dir = str(d)
        try:
            te.cal_auc() if shape == "ycb" else te.cal_lm_add(obj_id)
        finally:
            ev_mod.config.log_eval_dir, ev_mod.config_lm.log_eval_dir = prev
        (f,) = glob.glob(str(d / "*.pkl"))
        with open(f, "rb") as fh:
            pk.append(pickle.load(fh))
    for key in ("add_auc_lst", "adds_auc_lst", "add_s_auc_lst"):
        assert np.abs(np.asarray(pk[1][key], np.float64) - np.asarray(pk[0][key], np.float64)).max() <= 1e-6, key
