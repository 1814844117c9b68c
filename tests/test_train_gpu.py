"""pvn3d_train_targets, train_batch and the loss kernels (FocalLoss, OFLoss, PVN3DLoss) on the GPU: against the goldens
recorded from the reference's get_item and lib/loss.py (tests/golden/train_cases.npz), against the float64
restatements of tests/train_ref.py at the training shape, and against the reference's own lib/loss.py where the
reference Python is staged (oracle/_ref/py).

Bounds (u = 2^-24, the float32 unit roundoff):
  * targets: each output is float32(x) of a float64 x; the kernel's float64 x may differ from numpy's by a few float64
    ulps (summation order / FMA of the 3-term dot product), which can move the float32 rounding by at most 1 ulp.
  * focal: a row's log_softmax takes C exps, one log and a few subtractions, each with a relative error of a few u
    of the row's exponent arguments, so |err(row loss)| <= 256 u (1 + |logpt|), and the mean inherits the mean of that.
    Each gradient element is (g/M) f (delta - p) with f, p in [0, 1]: |err| <= 256 u (g/M) (1 + |logpt|).
  * OF: the loss is a float32 sum of 3n terms in a 3-deep per-thread chain, a 5-level warp tree and a 4-way block sum
    (float64 across blocks): |err| <= 32 u sum(w |diff|) / den + 2 u |loss|.  The gradient is +-(g/den) or 0 with
    exact signs (a float32 difference has the sign of the exact one): |err| <= 2 u |ref|.
"""
import os

import numpy as np
import pytest
import torch

import train_ref as R
from helpers import load_reference_python
from pvn3d_b200 import compat, fixtures
from pvn3d_b200 import train_utils as T
from pvn3d_b200.frame_input import FrameInputBuilder

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


@pytest.fixture(scope="module")
def gold(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "train_cases.npz")))


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
    return np.abs(ia - ib)


def _check_targets(got, want, what):
    equal = 0
    total = 0
    for g, w, name in zip(got, want, ("kp_targ_ofst", "ctr_targ_ofst", "kp3ds", "ctr3ds")):
        g = g.cpu().numpy()
        assert g.shape == w.shape, (what, name)
        d = _ulps(g, w)
        assert d.max() <= 1, f"{what} {name}: {int(d.max())} ulps"
        equal += int((d == 0).sum())
        total += d.size
    print(f"{what}: {equal}/{total} bit-equal, the rest within 1 ulp")
    return equal, total


def test_targets_match_get_item(cuda_dev, gold):
    tt = T.TrainTargets(kp_table=gold["tgt_kp_table"], ctr_table=gold["tgt_ctr_table"], device=cuda_dev)
    pcld = torch.from_numpy(gold["tgt_pcld"]).to(cuda_dev)
    lab = torch.from_numpy(gold["tgt_labels"]).to(cuda_dev)
    ids = torch.from_numpy(gold["tgt_cls_ids"]).to(cuda_dev)        # get_item's [B,22,1] int64
    rts = torch.from_numpy(gold["tgt_rts64"]).to(cuda_dev)
    got = tt.compute(pcld, lab, ids, rts)
    # the goldens keep get_item's kp_targ_ofst at every ROW_STRIDE-th point and as a SHA-256 of the whole tensor
    rows = (got[0][:, ::R.ROW_STRIDE],) + tuple(got[1:])
    want = [gold[n] for n in ("tgt_kp_targ_ofst_rows", "tgt_ctr_targ_ofst", "tgt_kp3ds", "tgt_ctr3ds")]
    eq, tot = _check_targets(rows, want, "get_item goldens")
    assert eq >= 0.99 * tot
    same = R.digest(got[0].cpu().numpy()) == str(gold["tgt_kp_targ_ofst_sha256"])
    print("whole kp_targ_ofst bit-equal to get_item's:", same)
    full = R.targets_ref(gold["tgt_pcld"], gold["tgt_labels"], gold["tgt_slot_ids"], gold["tgt_rts64"],
                         gold["tgt_kp_table"], gold["tgt_ctr_table"])      # bit-equal to get_item (host test)
    _check_targets(got, full, "get_item goldens, every point")
    # the fixtures' YCB tables are the ones get_item loads
    t = fixtures.mesh_kps_table_ycb()
    assert np.array_equal(t[1:, :8], gold["tgt_kp_table"][1:]) and np.array_equal(t[1:, 8], gold["tgt_ctr_table"][1:])
    again = tt.compute(pcld, lab, ids, rts)
    assert all(torch.equal(a, b) for a, b in zip(got, again))


def test_targets_k16_and_out_of_range_ids(cuda_dev):
    rng = np.random.default_rng(3)
    b, n, s, n_cls, k = 3, 5000, 22, 22, 16
    kp = rng.normal(0, 0.05, (n_cls, k, 3)).astype(np.float32)
    ctr = rng.normal(0, 0.02, (n_cls, 3)).astype(np.float32)
    pcld = rng.normal(0, 0.3, (b, n, 3)).astype(np.float32) + np.float32([0, 0, 1])
    labels = rng.integers(-3, 30, (b, n)).astype(np.int32)
    labels[:, :10] = [-1, 0, 21, 22, 25, 200, -(1 << 31), (1 << 31) - 1, 1, 2]
    ids = np.zeros((b, s), np.int32)
    ids[0, :6] = [1, 2, 3, 2, 21, 5]
    ids[1, :7] = [4, 0, 6, 30, -2, 22, 4]          # 0 in the middle, ids past the table, a repeated class
    ids[2, :3] = [1 << 30, 7, 8]
    rts = np.zeros((b, s, 3, 4))
    for f in range(b):
        for i in range(s):
            q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
            rts[f, i] = np.concatenate([q, rng.normal(0, 0.3, (3, 1))], 1)
    tt = T.TrainTargets(kp_table=kp, ctr_table=ctr, device=cuda_dev)
    d = lambda a: torch.from_numpy(a).to(cuda_dev)  # noqa: E731
    got = tt.compute(d(pcld), d(labels), d(ids), d(rts))
    want = R.targets_ref(pcld, labels, ids, rts, kp, ctr)
    _check_targets(got, want, "K=16, out-of-range ids and labels")
    for f, i in ((1, 1), (1, 3), (1, 4), (1, 5), (2, 0)):     # empty and out-of-range slots: zero kp3ds / ctr3ds
        assert float(got[2][f, i].abs().max()) == 0 and float(got[3][f, i].abs().max()) == 0
    # LineMOD: S = 2, cls_ids = [1, 0]
    lm = T.TrainTargets.linemod(next(iter(fixtures.lm_obj_dict().values())), device=cuda_dev)
    lab = (rng.random((2, 3000)) < 0.4).astype(np.int32)
    ids2 = np.array([[1, 0], [1, 0]], np.int32)
    got = lm.compute(d(pcld[:2, :3000]), d(lab), d(ids2), d(rts[:2, :2]))
    want = R.targets_ref(pcld[:2, :3000], lab, ids2, rts[:2, :2], lm.kp_table.cpu().numpy(), lm.ctr_table.cpu().numpy())
    _check_targets(got, want, "LineMOD")


def _frames(b, h=480, w=640, seed=0):
    return R.raw_frames(b, h, w, seed, sparse=(1,))       # frame 1: 300 valid pixels, ok = 0


def test_train_batch_end_to_end(cuda_dev):
    b, n = 3, 12288
    depth, K, cs, rgb, label, ids, rts = (torch.from_numpy(a).to(cuda_dev) for a in _frames(b))
    builder = FrameInputBuilder(b, n, device=cuda_dev)
    targets = T.TrainTargets(device=cuda_dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = T.train_batch(builder, targets, depth, K, cs, rgb, label, ids, rts, seed=11)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    rgb_o, pcld, cld, choose, kp_t, ctr_t, ids_o, rts_o, lab, kp3, ctr3, ok = out
    shapes = [(b, 3, 480, 640), (b, n, 3), (b, n, 9), (b, 1, n), (b, n, 8, 3), (b, n, 3), (b, 22, 1), (b, 22, 3, 4),
              (b, n), (b, 22, 8, 3), (b, 22, 3), (b,)]
    dtypes = [torch.float32] * 3 + [torch.int64] + [torch.float32] * 2 + [torch.int64, torch.float32, torch.int64] + \
        [torch.float32] * 2 + [torch.uint8]
    for t, s, dt in zip(out, shapes, dtypes):
        assert tuple(t.shape) == s and t.dtype == dt and t.device == cuda_dev
    assert ok.tolist() == [1, 0, 1]
    flat = label.reshape(b, -1)
    assert torch.equal(lab, torch.gather(flat, 1, choose[:, 0]).to(torch.int64) * ok[:, None].long())
    t = fixtures.mesh_kps_table_ycb()
    want = R.targets_ref(pcld.cpu().numpy(), lab.cpu().numpy(), ids.cpu().numpy(),
                         rts.cpu().numpy(), t[:, :8], t[:, 8])
    _check_targets((kp_t, ctr_t, kp3, ctr3), want, "train_batch")
    assert float(kp_t[1].abs().max()) == 0 and float(ctr_t[1].abs().max()) == 0 and int(lab[1].abs().max()) == 0
    assert (kp_t[0].abs().sum((1, 2)) > 0).sum() == (lab[0] > 0).sum()


# --- losses -------------------------------------------------------------------------------------------------------

def _training_inputs(dev, b=24, n=12288, c=22, k=8, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    seg = (torch.randn(b, n, c, generator=g) * 3).to(dev)
    labels = torch.randint(0, c, (b, n), generator=g)
    labels[torch.rand(b, n, generator=g) < 0.7] = 0
    kp = (torch.randn(b, k, n, 3, generator=g) * 0.1).to(dev)
    ctr = (torch.randn(b, 1, n, 3, generator=g) * 0.1).to(dev)
    kt = (torch.randn(b, n, k, 3, generator=g) * 0.1).to(dev)
    ct = (torch.randn(b, n, 3, generator=g) * 0.1).to(dev)
    return kp, seg, ctr, kt, ct, labels.to(dev)


def _focal_bounds(z, t, g_over_m, mask=None):
    logpt = torch.log_softmax(torch.as_tensor(z, dtype=torch.float64), 1).gather(1, torch.as_tensor(t)[:, None])[:, 0]
    scale = (1 + logpt.abs()).numpy()
    if mask is not None:
        scale = np.where(mask, scale, 0)
        m = max(int(mask.sum()), 1)
    else:
        m = len(scale)
    return 256 * U * scale.sum() / m + 1e-30, 256 * U * g_over_m * scale[:, None] + 1e-30


def test_losses_against_goldens(cuda_dev, gold):
    for i in range(int(gold["n_focal"])):
        z, t, gamma = gold[f"focal{i}_z"].astype(np.float32), gold[f"focal{i}_t"], float(gold[f"focal{i}_gamma"])
        x = torch.from_numpy(z).to(cuda_dev).requires_grad_(True)
        loss = T.FocalLoss(gamma=gamma)(x, torch.from_numpy(t).to(cuda_dev))
        loss.backward()
        lb, gb = _focal_bounds(z, t, 1.0 / len(t))
        assert abs(float(loss) - float(gold[f"focal{i}_loss"])) <= lb, i
        assert (np.abs(x.grad.cpu().numpy() - gold[f"focal{i}_grad"]) <= gb).all(), i
    for i in range(int(gold["n_of"])):
        pred = torch.from_numpy(gold[f"of{i}_pred"]).to(cuda_dev).requires_grad_(True)
        targ = torch.from_numpy(gold[f"of{i}_targ"]).to(cuda_dev)
        lab = torch.from_numpy(gold[f"of{i}_labels"]).to(cuda_dev)
        g = torch.from_numpy(gold[f"of{i}_g"]).float().to(cuda_dev)
        loss = T.OFLoss()(pred, targ, lab)
        (loss * g).sum().backward()
        _check_of(loss, pred.grad, gold[f"of{i}_pred"], gold[f"of{i}_targ"], gold[f"of{i}_labels"],
                  gold[f"of{i}_loss"], gold[f"of{i}_grad"], g.cpu().numpy())


def _check_of(loss, grad, pred, targ, labels, want_loss, want_grad, g):
    bs, k, n, _ = pred.shape
    t = np.asarray(targ, np.float64).reshape(bs, n, k, 3).transpose(0, 2, 1, 3)
    w = (np.asarray(labels).reshape(bs, 1, n, 1) > 0)
    sabs = (w * np.abs(np.asarray(pred, np.float64) - t)).sum((2, 3))
    den = w.sum((2, 3)).astype(np.float32) + np.float32(1e-3)
    bound = 32 * U * sabs / den + 2 * U * np.abs(want_loss)
    assert (np.abs(loss.detach().cpu().numpy() - want_loss) <= bound).all()
    assert (np.abs(grad.cpu().numpy() - want_grad) <= 2 * U * np.abs(want_grad)).all()


def test_pvn3d_loss_at_training_shape(cuda_dev):
    kp, seg, ctr, kt, ct, labels = _training_inputs(cuda_dev)
    ok = torch.ones(24, dtype=torch.uint8, device=cuda_dev)
    ok[[3, 17]] = 0
    labels[[3, 17]] = 0              # FrameInputBuilder zero-fills ok = 0 frames: their labels are 0
    crit = T.PVN3DLoss()

    def run(module, ok_):
        ins = [t.clone().requires_grad_(True) for t in (kp, seg, ctr)]
        loss, parts, acc = module(ins[0], ins[1], ins[2], kt, ct, labels, ok_)
        loss.backward()
        return loss.detach(), parts.detach(), acc, [t.grad for t in ins]

    for ok_ in (None, ok):
        loss, parts, acc, grads = run(crit, ok_)
        okn = None if ok_ is None else ok_.cpu().numpy()
        rl, rp, ra, rdk, rds, rdc = R.pvn3d_loss_ref(kp.cpu().numpy(), seg.cpu().numpy(), ctr.cpu().numpy(),
                                                     kt.cpu().numpy(), ct.cpu().numpy(), labels.cpu().numpy(), okn)
        z = seg.reshape(-1, 22).cpu().numpy()
        t = labels.reshape(-1).cpu().numpy()
        mask = None if okn is None else np.repeat(okn != 0, 12288)
        m = len(t) if mask is None else int(mask.sum())
        lb, gb = _focal_bounds(z, t, 2.0 / m, mask)
        assert abs(float(parts[0]) - rp[0]) <= lb
        assert (np.abs(grads[1].cpu().numpy().reshape(-1, 22) - rds.reshape(-1, 22)) <= gb).all()
        assert abs(float(parts[1]) - rp[1]) <= 1e-5 * rp[1] and abs(float(parts[2]) - rp[2]) <= 1e-5 * rp[2]
        assert abs(float(loss) - rl) <= 2 * lb + 1e-5 * (rp[1] + rp[2])
        assert abs(float(acc) - ra) <= 2 * U
        assert (np.abs(grads[0].cpu().numpy() - rdk) <= 2 * U * np.abs(rdk)).all()
        assert (np.abs(grads[2].cpu().numpy() - rdc) <= 2 * U * np.abs(rdc)).all()
        if ok_ is not None:
            assert float(grads[1][[3, 17]].abs().max()) == 0
        # bit-identical on a repeat call and through nn.DataParallel on one device
        again = run(crit, ok_)
        dp = run(torch.nn.DataParallel(crit, device_ids=[cuda_dev.index]), ok_)
        for other in (again, dp):
            assert torch.equal(other[0], loss) and torch.equal(other[1], parts) and torch.equal(other[2], acc)
            assert all(torch.equal(a, b) for a, b in zip(other[3], grads))
    # PVN3DLoss = 2 FocalLoss(2) + sum OFLoss(kp) + sum OFLoss(ctr)
    focal = T.FocalLoss(gamma=2)(seg.view(labels.numel(), -1), labels.view(-1))
    kpl = T.OFLoss()(kp, kt, labels).sum()
    ctl = T.OFLoss()(ctr, ct, labels).sum()
    loss, parts, _, _ = run(crit, None)
    assert torch.equal(parts[0], focal) and torch.allclose(parts[1:], torch.stack([kpl, ctl]), rtol=1e-6, atol=0)
    assert torch.allclose(loss, 2 * focal + kpl + ctl, rtol=1e-6, atol=0)
    # no ok frame: loss, parts[0], acc and the gradient are 0
    none = torch.zeros(24, dtype=torch.uint8, device=cuda_dev)
    zl = torch.zeros_like(labels)
    x = seg.clone().requires_grad_(True)
    loss, parts, acc = crit(kp, x, ctr, kt, ct, zl, none)
    loss.backward()
    assert float(loss) == 0 and float(acc) == 0 and float(x.grad.abs().max()) == 0


def test_focal_nan_rows_nchw_and_sum(cuda_dev):
    rng = np.random.default_rng(5)
    z = rng.normal(0, 2, (4, 22, 8, 16)).astype(np.float32)        # N,C,H,W: reshaped to N*H*W rows in place
    t = rng.integers(0, 22, (4, 8, 16))
    x = torch.from_numpy(z).to(cuda_dev).requires_grad_(True)
    for mean in (True, False):
        x.grad = None
        loss = T.FocalLoss(gamma=2, size_average=mean)(x, torch.from_numpy(t).to(cuda_dev))
        loss.backward()
        rows = z.transpose(0, 2, 3, 1).reshape(-1, 22)
        rl, rg = R.focal_ref(rows, t.reshape(-1), 2.0, mean=mean)
        lb, gb = _focal_bounds(rows, t.reshape(-1), 1.0 / len(rows) if mean else 1.0)
        assert abs(float(loss) - rl) <= (lb if mean else lb * len(rows))
        got = x.grad.cpu().numpy().transpose(0, 2, 3, 1).reshape(-1, 22)
        assert (np.abs(got - rg) <= gb).all()
    # a target outside [0, C): that row's loss and gradient are NaN, no other row changes, no sync
    tt = torch.from_numpy(t.reshape(-1)).to(cuda_dev)
    tt[[5, 77]] = torch.tensor([22, -1], device=cuda_dev)
    x2 = torch.from_numpy(z.transpose(0, 2, 3, 1).reshape(-1, 22).copy()).to(cuda_dev).requires_grad_(True)
    loss = T.FocalLoss(gamma=2)(x2, tt)
    loss.backward()
    g = x2.grad.cpu().numpy()
    assert np.isnan(float(loss))
    assert np.isnan(g[[5, 77]]).all() and np.isfinite(np.delete(g, [5, 77], 0)).all()
    # float64 and bfloat16 inputs are upcast; the gradient returns in the input's dtype
    xd = torch.from_numpy(z).double().to(cuda_dev).requires_grad_(True)
    T.FocalLoss(gamma=2)(xd, torch.from_numpy(t).to(cuda_dev)).backward()
    assert xd.grad.dtype == torch.float64


def test_against_staged_reference_loss(cuda_dev):
    ref = load_reference_python()
    if ref is None:
        pytest.skip("reference Python not staged under oracle/_ref/py")
    import importlib

    lib_loss = importlib.import_module("lib.loss")
    kp, seg, ctr, kt, ct, labels = _training_inputs(cuda_dev, seed=4)
    pairs = [(lib_loss.FocalLoss(gamma=2), T.FocalLoss(gamma=2), (seg.view(labels.numel(), -1), labels.view(-1))),
             (lib_loss.OFLoss(), T.OFLoss(), (kp, kt, labels)), (lib_loss.OFLoss(), T.OFLoss(), (ctr, ct, labels))]
    for theirs, ours, args in pairs:
        xs = [args[0].clone().requires_grad_(True) for _ in range(2)]
        a = theirs(xs[0], *args[1:])
        b = ours(xs[1], *args[1:])
        a.sum().backward()
        b.sum().backward()
        # both are float32 evaluations of the same function: within the sum of the two float32 bounds above
        assert torch.allclose(b, a, rtol=2e-5, atol=0), type(ours).__name__
        assert torch.allclose(xs[1].grad, xs[0].grad, rtol=1e-4, atol=1e-6 * float(xs[0].grad.abs().max()))


def test_compat_patch_loss(cuda_dev):
    ref = load_reference_python()
    if ref is None:
        pytest.skip("reference Python not staged under oracle/_ref/py")
    import importlib
    import sys

    lib_loss = importlib.import_module("lib.loss")
    orig = lib_loss.FocalLoss, lib_loss.OFLoss
    try:
        root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "py")
        compat.install(root)
        assert (lib_loss.FocalLoss, lib_loss.OFLoss) == orig
        compat.install(root, patch_loss=True)
        assert lib_loss.FocalLoss is T.FocalLoss and lib_loss.OFLoss is T.OFLoss
        fake = type(sys)("train.train_ycb_pvn3d")
        fake.FocalLoss, fake.OFLoss = orig
        sys.modules["train.train_ycb_pvn3d"] = fake
        compat.install(root, patch_loss=True)
        assert fake.FocalLoss is T.FocalLoss and fake.OFLoss is T.OFLoss
    finally:
        lib_loss.FocalLoss, lib_loss.OFLoss = orig
        sys.modules.pop("train.train_ycb_pvn3d", None)
