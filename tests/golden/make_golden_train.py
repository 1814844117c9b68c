"""Record get_item's training targets and lib/loss.py's losses from the REFERENCE ITSELF on the CPU (build container
only).

    python tests/golden/make_golden_train.py          # writes train_cases.npz + make_golden_train.log

Targets: the unmodified YCB_Dataset('test').get_item (ycb_dataset.py:179-309) on synthetic 480x640 frames written to a
temporary root as depth / label / colour PNGs and a meta.mat.  The import shims of pvn3d_b200.compat stub `pcl`,
get_normal is replaced by zeros (normals are not part of the targets), np.random is seeded before every frame (the
point subset comes from np.random.shuffle), and config.n_sample_points is set to N_POINTS = 2048 instead of 12288 so
that the npz stays small (get_item's target code does not depend on it).  The frames hold several objects, a class
listed twice in meta (the last slot wins), a label with no meta entry, and one frame with fewer than N_POINTS valid
pixels ('wrap' pad).  Recorded: the float64 meta slots (slot_ids, rts64) and all 11 outputs of every frame (tgt_*),
compactly: kp_targ_ofst as its SHA-256 and every 8th point, cld_rgb_nrm as its SHA-256 (it is rebuilt from pcld, the
colours and choose), the colours as uint8.

Losses: the unmodified lib/loss.py FocalLoss / OFLoss in float64 with autograd on seeded float32-representable inputs:
C in {2, 22}, K in {8, 16}, logits of +-80, tied logits, pt -> 1, a frame with no labelled point, gamma in {0, 2}.
Recorded: inputs, losses and gradients (focal_*, of_*).

While recording, tests/train_ref.py is checked against every reference value (targets bit for bit, losses to 1e-12
relative) and every mutant of train_ref.MUTANTS must differ from the reference on some case; a mismatch aborts.
"""
import importlib.util
import os
import sys
import tempfile
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
REF = os.environ.get("PVN3D_REFERENCE", "/root/reference/pvn3d")

from PIL import Image  # noqa: E402
import scipy.io as scio  # noqa: E402

from pvn3d_b200 import compat, synth  # noqa: E402
from oracle import ext_cpu  # noqa: E402
import train_ref as R  # noqa: E402

if not hasattr(np, "bool"):
    np.bool = bool  # the reference's ip_basic predates numpy 1.24
compat.install_import_shims()
sys.modules["lib.pointnet2_utils._ext"] = ext_cpu
sys.path.insert(0, REF)
LOG = []
N_POINTS = 2048      # config.n_sample_points for the recorded frames (12288 in the reference's config): keeps the npz small


def log(msg):
    print(msg)
    LOG.append(msg)


def _pose(rng):
    r = synth._haar_rotation(rng)
    t = rng.uniform([-0.15, -0.1, 0.7], [0.15, 0.1, 1.0])
    return np.concatenate([r, t[:, None]], 1)


def _frame(rng, kind):
    """depth (uint16, factor 10000), label (uint8), colour, meta cls_indexes and the slots' poses"""
    h, w = 480, 640
    yy, xx = np.mgrid[0:h, 0:w]
    depth = (9000 + 800 * np.sin(xx / 90.0) + 500 * np.cos(yy / 70.0)).astype(np.float64)
    label = np.zeros((h, w), np.uint8)
    if kind == "objects":           # classes 1, 5 (twice in meta), 12 and 21, plus 7 which has no meta entry
        boxes = {1: (40, 200, 60, 260), 5: (220, 400, 80, 300), 12: (100, 300, 350, 520), 21: (330, 470, 420, 620),
                 7: (10, 90, 500, 630)}
        meta_ids = [1, 5, 12, 5, 21]
    elif kind == "dense":          # many classes side by side
        boxes = {c: (20 + 110 * ((c - 1) // 5), 120 + 110 * ((c - 1) // 5), 20 + 120 * ((c - 1) % 5),
                     130 + 120 * ((c - 1) % 5)) for c in range(2, 20, 2)}
        meta_ids = list(range(2, 20, 2))
    else:                          # "sparse": a 6x10 patch of depth only; fill_missing grows it to about 1600
        boxes = {3: (185, 203, 285, 325), 9: (203, 221, 285, 325)}     # valid pixels, fewer than N_POINTS
        meta_ids = [9, 3]
        keep = np.zeros((h, w), bool)
        keep[200:206, 300:310] = True
        depth[~keep] = 0
    for c, (y0, y1, x0, x1) in boxes.items():
        label[y0:y1, x0:x1] = c
        box = depth[y0:y1, x0:x1]
        box[box > 0] -= 600 + 40 * c            # objects in front of the wall; holes stay holes
    if kind != "sparse":
        depth[rng.random((h, w)) < 0.02] = 0       # missing pixels: fill_missing's work
    colour = np.stack([(xx + 2 * yy + 40 * c) % 256 for c in range(3)], -1).astype(np.uint8)
    poses = np.stack([_pose(rng) for _ in meta_ids], 2)      # [3,4,n] float64, as meta['poses']
    return depth.astype(np.uint16), label, colour, np.array(meta_ids, np.float64)[:, None], poses


def record_targets(out):
    cwd = os.getcwd()
    os.chdir(REF)          # YCB_Dataset reads its list files relative to the working directory
    try:
        spec = importlib.util.spec_from_file_location(
            "ref_ycb_dataset", os.path.join(REF, "datasets", "ycb", "ycb_dataset.py"))
        ycb = importlib.util.module_from_spec(spec)   # by path: an installed `datasets` package shadows the folder
        spec.loader.exec_module(ycb)
        ds = ycb.YCB_Dataset("test")
    finally:
        os.chdir(cwd)
    ds.get_normal = lambda cld: np.zeros((len(cld), 3), np.float32)
    ycb.config.n_sample_points = N_POINTS     # read by get_item at call time (ycb_dataset.py:227-245)
    kinds = ["objects", "dense", "sparse"]
    rng = np.random.default_rng(2024)
    names = ["rgb", "pcld", "cld_rgb_nrm", "choose", "kp_targ_ofst", "ctr_targ_ofst", "cls_ids", "RTs", "labels",
             "kp3ds", "ctr3ds"]
    rec = {n: [] for n in names}
    slots_ids, slots_rt = [], []
    with tempfile.TemporaryDirectory() as root:
        ds.root = root
        os.makedirs(os.path.join(root, "data_syn"))
        for i, kind in enumerate(kinds):
            depth, label, colour, ids, poses = _frame(rng, kind)
            item = f"data_syn/{i:06d}"
            Image.fromarray(depth).save(os.path.join(root, item + "-depth.png"))
            Image.fromarray(label).save(os.path.join(root, item + "-label.png"))
            Image.fromarray(colour).save(os.path.join(root, item + "-color.png"))
            scio.savemat(os.path.join(root, item + "-meta.mat"),
                         {"cls_indexes": ids, "poses": poses, "factor_depth": np.array([[10000.0]])})
            np.random.seed(100 + i)
            t0 = time.perf_counter()
            data = ds.get_item(item)
            dt = time.perf_counter() - t0
            assert data is not None, f"get_item dropped frame {i}"
            data = [d.numpy() for d in data]
            n_valid = int((np.asarray(Image.open(os.path.join(root, item + "-depth.png"))) > 0).sum())
            log(f"frame {i} ({kind}): {len(ids)} meta slots {ids[:, 0].astype(int).tolist()}, {n_valid} valid depth "
                f"pixels before fill, get_item {dt * 1e3:.0f} ms (fill_missing included, normals stubbed)")
            for n, d in zip(names, data):
                rec[n].append(d)
            n_used = len(np.unique(data[names.index("choose")]))
            assert (n_used < N_POINTS) == (kind == "sparse"), f"frame {i}: {n_used} distinct points"
            sid = np.zeros(22, np.int32)
            sid[:len(ids)] = ids[:, 0]
            srt = np.zeros((22, 3, 4))
            srt[:len(ids)] = poses.transpose(2, 0, 1)
            slots_ids.append(sid)
            slots_rt.append(srt)
    for n in names:
        out["tgt_" + n] = np.stack(rec[n])
    # compact storage (the tests rebuild or hash what is not stored in full; see tests/test_train_host.py):
    # integer colours as uint8, choose as int32, kp_targ_ofst as its SHA-256 plus every ROW_STRIDE-th row,
    # cld_rgb_nrm as its SHA-256 (it is pcld, the colours at choose and the stubbed zero normals)
    for n, dt in (("rgb", np.uint8), ("choose", np.int32), ("labels", np.int32), ("cls_ids", np.int32)):
        assert np.array_equal(out["tgt_" + n], out["tgt_" + n].astype(dt)), n
        out["tgt_" + n] = out["tgt_" + n].astype(dt)
    assert np.array_equal(R.cld_rgb_nrm_of(out["tgt_pcld"], out["tgt_rgb"], out["tgt_choose"]), out["tgt_cld_rgb_nrm"])
    for n in ("kp_targ_ofst", "cld_rgb_nrm"):
        out[f"tgt_{n}_sha256"] = np.array(R.digest(out["tgt_" + n]))
    full_kp = out.pop("tgt_kp_targ_ofst")
    out.pop("tgt_cld_rgb_nrm")
    out["tgt_kp_targ_ofst_rows"] = full_kp[:, ::R.ROW_STRIDE]
    out["tgt_slot_ids"] = np.stack(slots_ids)
    out["tgt_rts64"] = np.stack(slots_rt)
    cls_lst = ds.cls_lst
    kp = np.zeros((22, 8, 3), np.float32)
    ctr = np.zeros((22, 3), np.float32)
    for c in range(1, 22):
        kp[c] = ycb.bs_utils.get_kps(cls_lst[c - 1], kp_type="farthest", ds_type="ycb")
        ctr[c] = ycb.bs_utils.get_ctr(cls_lst[c - 1])
    out["tgt_kp_table"], out["tgt_ctr_table"] = kp, ctr
    # the restatement reproduces every target bit for bit; first-slot-wins does not
    want = R.targets_ref(out["tgt_pcld"], out["tgt_labels"], out["tgt_slot_ids"], out["tgt_rts64"], kp, ctr)
    got = [full_kp, out["tgt_ctr_targ_ofst"], out["tgt_kp3ds"], out["tgt_ctr3ds"]]
    for w, g, n in zip(want, got, ("kp_targ_ofst", "ctr_targ_ofst", "kp3ds", "ctr3ds")):
        assert np.array_equal(w, g), f"train_ref.targets_ref differs from get_item on {n}"
    bad = R.targets_ref(out["tgt_pcld"], out["tgt_labels"], out["tgt_slot_ids"], out["tgt_rts64"], kp, ctr,
                        mutant="first_slot_wins")
    assert not np.array_equal(bad[0], got[0]), "first_slot_wins not told apart"
    n_lab = (out["tgt_labels"] > 0).sum(1)
    log(f"targets: {len(kinds)} frames, labelled points per frame {n_lab.tolist()}; train_ref bit-equal, "
        "first_slot_wins told apart")


def _logits(rng, m, c, kind):
    z = rng.normal(0, 3, (m, c)).astype(np.float32)
    t = rng.integers(0, c, m)
    if kind == "big":
        z = rng.choice(np.float32([-80, 80, 0, 79.5]), (m, c)).astype(np.float32)
    elif kind == "ties":
        z = np.round(z).astype(np.float32)
        z[: m // 4] = 1.0
    elif kind == "sure":              # pt -> 1 and pt == 1 in float64: (1-pt)^gamma -> 0 (0^0 = 1 at gamma = 0)
        z[np.arange(m), t] = np.float32(40.0)
        z[: m // 8, :] = -np.float32(800.0)
        z[np.arange(m // 8), t[: m // 8]] = np.float32(800.0)
    return z, t


def record_losses(out):
    from lib.loss import FocalLoss, OFLoss

    rng = np.random.default_rng(7)
    seen = {m: False for m in ("pt_not_detached", "den_3x")}
    fi = 0
    for c in (2, 22):
        for kind in ("plain", "big", "ties", "sure"):
            for gamma in (0, 2):
                z, t = _logits(rng, 96, c, kind)
                x = torch.from_numpy(z.astype(np.float64)).requires_grad_(True)
                loss = FocalLoss(gamma=gamma)(x, torch.from_numpy(t))
                loss.backward()
                lv, gv = float(loss), x.grad.numpy()
                rl, rg = R.focal_ref(z, t, gamma)
                assert abs(rl - lv) <= 1e-12 * abs(lv) + 1e-300 and np.allclose(rg, gv, rtol=1e-12, atol=1e-300), \
                    f"focal_ref differs from FocalLoss (C={c}, {kind}, gamma={gamma})"
                ml, mg = R.focal_ref(z, t, gamma, mutant="pt_not_detached")
                if gamma and not np.allclose(mg, gv, rtol=1e-6, atol=1e-12):
                    seen["pt_not_detached"] = True
                for k, v in dict(z=z, t=t, gamma=np.float64(gamma), loss=np.float64(lv), grad=gv).items():
                    out[f"focal{fi}_{k}"] = v
                fi += 1
    oi = 0
    for k in (8, 16):
        for empty in (False, True):
            bs, n = 3, 48
            pred = rng.normal(0, 0.1, (bs, k, n, 3)).astype(np.float32)
            targ = rng.normal(0, 0.1, (bs, n, k, 3)).astype(np.float32)
            labels = rng.integers(0, 4, (bs, n)) * (rng.random((bs, n)) < 0.6)
            if empty:
                labels[1] = 0            # a frame with no labelled point: loss 0, gradient 0
            pred[0, 0, :5] = targ[0, :5, 0]   # zero differences: torch.abs's gradient 0
            g = rng.normal(0, 1, (bs, k))
            x = torch.from_numpy(pred.astype(np.float64)).requires_grad_(True)
            loss = OFLoss()(x, torch.from_numpy(targ.astype(np.float64)), torch.from_numpy(labels))
            (loss * torch.from_numpy(g)).sum().backward()
            lv, gv = loss.detach().numpy(), x.grad.numpy()
            rl, rg = R.of_ref(pred, targ, labels, g)
            assert np.allclose(rl, lv, rtol=1e-12, atol=0) and np.allclose(rg, gv, rtol=1e-12, atol=0), \
                f"of_ref differs from OFLoss (K={k})"
            ml, _ = R.of_ref(pred, targ, labels, g, mutant="den_3x")
            if not np.allclose(ml, lv, rtol=1e-6):
                seen["den_3x"] = True
            for key, v in dict(pred=pred, targ=targ, labels=labels, g=g, loss=lv, grad=gv).items():
                out[f"of{oi}_{key}"] = v
            oi += 1
    assert all(seen.values()), f"mutants not told apart: {seen}"
    out["n_focal"], out["n_of"] = np.int64(fi), np.int64(oi)
    log(f"losses: {fi} FocalLoss cases (C 2/22, plain/+-80/ties/pt->1, gamma 0/2), {oi} OFLoss cases (K 8/16, one "
        "with an unlabelled frame); train_ref within 1e-12, pt_not_detached and den_3x told apart")


def main():
    out = {}
    record_targets(out)
    record_losses(out)
    np.savez_compressed(os.path.join(HERE, "train_cases.npz"), **out)
    with open(os.path.join(HERE, "make_golden_train.log"), "w") as f:
        f.write("\n".join(LOG) + "\n")


if __name__ == "__main__":
    main()
