"""`FramePoseSolver` on the bench's synthetic batches against a float64 composition of the reference's
cal_frame_poses (oracle/frame_poses_oracle.py, with the float64 mean-shift of tests/ms_f64.py in place of the
oracle's iterations).

Per frame: `present` and the class ids exact; the relabelled mask exact (after asserting that no point lies within
MARGIN of its radius threshold, or -- where a centre could take it -- of a tie between two centres, where the kernel's centres -- within the mean-shift
bound of the reference's -- could flip a verdict); every voted keypoint and centre within delta + bound of the
float64 star at T64 (the default mode is certified); every pose within the bound propagated from those keypoints:
|dR|_F <= 2 |A~|_F |dB|_F / (s_2 + s_3) + 1e-5 and |dt| <= |dB|_max + |dR|_F |mean A| + 1e-5, with A~ the centred
mesh keypoints and s the singular values of H.  A batch solve equals the per-frame solves bit for bit in the default
(certified) mode, and to 1e-5 in the all-seed modes, whose sweep variant follows the launch's total seed count.
"""
import numpy as np
import pytest
import torch

import ms_f64
from pvn3d_b200 import fixtures, synth
from pvn3d_b200.eval_utils import RADIUS, FramePoseSolver

pytestmark = pytest.mark.gpu
MARGIN = 1e-5      # m: > 2 (delta + bound) of a centre at bw = 0.08, plus float32 rounding of the distances


def _solver(shape, b, n, dev, mode="certified"):
    if shape == "linemod":
        return FramePoseSolver(b, n, 8, 2, fixtures.mesh_kps_table_lm(1), None, False, device=dev, mode=mode)
    return FramePoseSolver(b, n, 8, fixtures.YCB_N_CLASSES, fixtures.mesh_kps_table_ycb(),
                           fixtures.radius_thresholds_ycb(), True, device=dev, mode=mode)


def _solve(s, st, dev):
    args = [torch.from_numpy(np.ascontiguousarray(st[k])).to(dev) for k in ("pcld", "labels", "ctr_of", "kp_of")]
    return [t.clone().cpu().numpy() for t in s.solve(*args)]


def _ms(clouds, dev):
    return ms_f64.reference(clouds, RADIUS, 300, dev)


def reference_frame(pcld, mask, ctr_of, kp_of, shape, dev):
    """float64 composition of cal_frame_poses(_lm) for one frame -> dict"""
    n_cls = 2 if shape == "linemod" else fixtures.YCB_N_CLASSES
    t = torch.from_numpy
    pred_ctr = (t(pcld) - t(ctr_of)).numpy()                                         # :41
    pred_kp = (t(pcld)[None] - t(kp_of)).numpy()                                     # :42
    ids = np.unique(mask[mask > 0])
    if shape == "linemod":
        ids = ids[ids == 1]
    new_mask = mask.copy()
    if shape == "ycb" and len(ids):                                                 # :51-73
        ctr_refs = _ms([pred_ctr[mask == c] for c in ids], dev)
        ctrs = np.stack([r["traj"][r["T"]] for r in ctr_refs])
        d = np.linalg.norm(pred_ctr.astype(np.float64)[:, None, :] - ctrs[None], axis=2)
        order = np.argsort(d, axis=1, kind="stable")
        closest = ids[order[:, 0]]
        dmin = d[np.arange(len(d)), order[:, 0]]
        r08 = np.array([fixtures.radius_thresholds_ycb()[c] for c in closest], np.float64)
        # no verdict within MARGIN of flipping (exactly equal centres resolve by index in both)
        assert np.all(np.abs(dmin - r08)[mask > 0] > MARGIN), "a point at the radius threshold"
        if len(ids) > 1:
            # a near-tie matters only where either centre could take the point (beyond both radii, it stays put)
            d2 = d[np.arange(len(d)), order[:, 1]]
            r2 = np.array([fixtures.radius_thresholds_ycb()[c] for c in ids[order[:, 1]]], np.float64)
            reach = (mask > 0) & (dmin < np.maximum(r08, r2) + MARGIN)
            assert np.all((d2 - dmin)[reach] > MARGIN), "a point between two centres"
        upd = (mask > 0) & (dmin < r08)
        new_mask[upd] = closest[upd]
    cls_kps = np.zeros((n_cls, 9, 3))
    fits, slots = [], []
    for c in ids:
        m = new_mask == c
        if m.sum() < 1:
            continue
        _, mi, lab = ms_f64.exact_part(pred_ctr[m], RADIUS)
        fits.append(pred_ctr[m])
        slots.append((c, 8))
        for k in range(8):     # the YCB solver keeps the centre fit's inliers (:91-92); the LineMOD one all votes
            fits.append(pred_kp[k][m][lab] if shape == "ycb" else pred_kp[k][m])
            slots.append((c, k))
    refs = _ms(fits, dev)
    for (c, k), r in zip(slots, refs):
        cls_kps[c, k] = r["traj"][r["T"]]
    return dict(ids=ids, new_mask=new_mask, cls_kps=cls_kps, slots=slots, refs=refs)


def frame_failures(ref, b, st, out, shape, mesh, worst):
    """every check of frame b against its reference -> list of what failed (empty = all pass)"""
    poses, present, cls_kps, new_mask = out
    bad = []
    want_present = np.zeros(present.shape[1], np.uint8)
    want_present[np.unique(st["labels"][b][st["labels"][b] > 0])] = 1
    if shape == "linemod":
        want_present[2:] = 0
    if not np.array_equal(present[b], want_present):
        bad.append("present")
    if shape == "ycb" and not np.array_equal(new_mask[b], ref["new_mask"]):
        bad.append("new_mask")
    for c in ref["ids"]:
        if not (ref["new_mask"] == c).any():
            if not np.array_equal(poses[b, c], np.eye(4)[:3]):
                bad.append(f"identity pose {c}")
            continue
        err = np.linalg.norm(cls_kps[b, c].astype(np.float64) - ref["cls_kps"][c], axis=1)
        allow = np.array([ms_f64.centre_bound(x, RADIUS) + ms_f64.DELTA_REL * RADIUS for x in ref["cls_kps"][c]])
        worst["kps"] = max(worst["kps"], float((err / allow).max()))
        if not np.all(err <= allow):
            bad.append(f"keypoints {c}: {(err / allow).max():.3g}")
        A = mesh[c].astype(np.float64)
        Ac = A - A.mean(0)
        R64, t64, s = ref["pose"](A, ref["cls_kps"][c])
        dB = float(np.linalg.norm(allow))
        rb = (2 * np.linalg.norm(Ac) * dB / (s[1] + s[2]) if s[1] + s[2] > 0 else np.inf) + 1e-5
        tb = float(allow.max()) + rb * np.linalg.norm(A.mean(0)) + 1e-5
        dr = np.linalg.norm(poses[b, c, :, :3] - R64)
        dt = np.linalg.norm(poses[b, c, :, 3] - t64)
        worst["rot"] = max(worst["rot"], dr / rb)
        worst["trans"] = max(worst["trans"], dt / tb)
        if not (dr <= rb and dt <= tb):
            bad.append(f"pose {c}: {dr / rb:.3g} {dt / tb:.3g}")
    return bad


def check_batch(shape, st, out, frames_checked, dev, mesh):
    """asserts every check on the given frames; returns (worst ratios, {frame: reference})"""
    worst = dict(kps=0.0, rot=0.0, trans=0.0)
    refs = {}
    for b in frames_checked:
        ref = reference_frame(st["pcld"][b], st["labels"][b], st["ctr_of"][b], st["kp_of"][b], shape, dev)
        ref["pose"] = ms_f64.kabsch_f64
        bad = frame_failures(ref, b, st, out, shape, mesh, worst)
        assert not bad, (b, bad)
        refs[b] = ref
    return worst, refs


BENCH = {"ycb": dict(shape="ycb", batch=16, config_id=3, n=12288, kw={}, check=range(16)),
         "linemod": dict(shape="linemod", batch=32, config_id=2, n=12288, kw=dict(lm_obj_id=1), check=range(0, 32, 4)),
         "stress": dict(shape="ycb", batch=8, config_id=5, n=49152, kw=dict(n_instances=10), check=[0, 5])}


@pytest.mark.parametrize("cfg", list(BENCH))
def test_bench_batches_against_float64(cuda_dev, cfg):
    c = BENCH[cfg]
    frames = synth.make_batch(c["shape"], c["batch"], n_points=c["n"], config_id=c["config_id"], **c["kw"])
    st = synth.stack(frames)
    s = _solver(c["shape"], c["batch"], c["n"], cuda_dev)
    out = _solve(s, st, cuda_dev)
    mesh = fixtures.mesh_kps_table_lm(1) if c["shape"] == "linemod" else fixtures.mesh_kps_table_ycb()
    worst, refs = check_batch(c["shape"], st, out, list(c["check"]), cuda_dev, mesh)
    if cfg == "ycb":
        # the solver's last mean-shift call holds the B*n_cls centre fits, then keypoint fit (b*n_cls + c)*8 + k:
        # classes with votes have keypoint fits in the second 2048-fit launch chunk
        bc = c["batch"] * fixtures.YCB_N_CLASSES
        late = [(b, k) for b, r in refs.items() for k in r["ids"] if (r["new_mask"] == k).any()
                and bc + (b * fixtures.YCB_N_CLASSES + k) * 8 >= 2048]
        assert late, "no fit with votes in the second launch chunk"
    for k, v in worst.items():
        print(f"F64RATIO poses/{cfg}/{k} {v:.4f}")


def _add_class(st, b, idx, cls, vote, rng, noise):
    """points idx of frame b become class cls, voting for centre `vote` (+ noise) and its keypoints"""
    mesh = fixtures.mesh_kps_table_ycb()[cls].astype(np.float64)
    p = st["pcld"][b][idx].astype(np.float64)
    v = vote + rng.normal(0, noise, (len(idx), 3))
    st["labels"][b][idx] = cls
    st["ctr_of"][b][idx] = (p - v).astype(np.float32)
    for k in range(8):
        st["kp_of"][b][k][idx] = (p - (v + mesh[k] - mesh[8])).astype(np.float32)


def test_hand_built_batch(cuda_dev):
    """n = 12287; a class above 4096 votes; a 1-point class; a class the relabel pass empties; classes absent in
    some frames.  The checks are also run against wrong references, and each must be caught."""
    n = 12287
    f0 = synth.make_frame("linemod", n_points=n, seed=11, obj_frac=0.45, lm_obj_id=1)
    f1 = synth.make_frame("ycb", n_points=n, seed=12)
    st = synth.stack([f0, f1])
    lab = st["labels"]
    big = lab[0] == 1
    assert big.sum() > 4096
    lab[0][big] = 5
    bg = np.flatnonzero(~big)
    lab[0][bg[0]] = 7                            # a 1-point class
    # classes 10 and 11 vote 0.12 m apart; class 12's two points vote exactly at their centres, so its own centre
    # (the single mode between its two votes) is 6 cm from both and the relabel pass moves both points away.  The
    # three vote behind the background plane, beyond the box the outlier votes fill, so no other point joins 12.
    rng = np.random.default_rng(3)
    cA = np.array([0.35, 0.25, 1.6])
    assert cA[2] - 0.3 > st["pcld"][0][:, 2].max()
    cB = cA + [0.12, 0.0, 0.0]
    _add_class(st, 0, bg[10:310], 10, cA, rng, 0.003)
    _add_class(st, 0, bg[400:700], 11, cB, rng, 0.003)
    _add_class(st, 0, bg[[800, 801]], 12, np.stack([cA, cB]), rng, 0.0)
    assert set(np.unique(lab[0])) != set(np.unique(lab[1]))
    s = _solver("ycb", 2, n, cuda_dev)
    out = _solve(s, st, cuda_dev)
    mesh = fixtures.mesh_kps_table_ycb()
    worst, refs = check_batch("ycb", st, out, [0, 1], cuda_dev, mesh)
    r0 = refs[0]
    assert 12 in r0["ids"] and not (r0["new_mask"] == 12).any(), "class 12 must be emptied by the relabel pass"
    assert np.array_equal(out[0][0, 12], np.eye(4)[:3])
    assert (r0["new_mask"] == 7).sum() == 1, "the 1-point class keeps its point"
    assert (r0["new_mask"] == 5).sum() > 4096
    for k, v in worst.items():
        print(f"F64RATIO poses/hand/{k} {v:.4f}")
    # wrong references: no relabel pass, keypoints in the wrong order, R transposed
    wrongs = {"no_relabel": dict(r0, new_mask=st["labels"][0].copy()),
              "rolled_keypoints": dict(r0, cls_kps=np.concatenate([np.roll(r0["cls_kps"][:, :8], 1, 1),
                                                                   r0["cls_kps"][:, 8:]], 1)),
              "transposed_R": dict(r0, pose=lambda A, B: (lambda R, t, s_: (R.T, t, s_))(*ms_f64.kabsch_f64(A, B)))}
    for name, w in wrongs.items():
        bad = frame_failures(w, 0, st, out, "ycb", mesh, dict(kps=0.0, rot=0.0, trans=0.0))
        assert bad, f"the wrong reference {name} was not caught"


@pytest.mark.parametrize("mode", ["certified", "strict", "no_freeze", "early_exit"])
def test_batch_equals_per_frame(cuda_dev, mode):
    """certified (the default; one CTA per fit) is bit-identical; the all-seed modes pick their sweep variant from
    the launch's total seed count, so a fit's sums may round differently in a batch: there the masks are equal, the
    keypoints within twice the float64 bound (plus delta for the star's last steps) and the poses to 1e-5"""
    frames = synth.make_batch("ycb", 12, n_points=4096, config_id=3)
    st = synth.stack(frames)
    whole = _solve(_solver("ycb", 12, 4096, cuda_dev, mode), st, cuda_dev)
    one = _solver("ycb", 1, 4096, cuda_dev, mode)
    for b in range(12):
        single = _solve(one, {k: v[b:b + 1] for k, v in st.items()}, cuda_dev)
        if mode == "certified":
            for w, x in zip(whole, single):
                assert np.array_equal(w[b], x[0]), (mode, b)
            continue
        assert np.array_equal(whole[1][b], single[1][0]) and np.array_equal(whole[3][b], single[3][0]), (mode, b)
        kw, ks = whole[2][b].astype(np.float64), single[2][0].astype(np.float64)
        allow = np.array([[2 * ms_f64.centre_bound(x, RADIUS) + ms_f64.DELTA_REL * RADIUS for x in row] for row in ks])
        assert np.all(np.linalg.norm(kw - ks, axis=-1) <= allow), (mode, b)
        assert np.abs(whole[0][b] - single[0][0]).max() <= 1e-5, (mode, b)
