"""csrc/train.cu's losses and targets at their edges, against the float64 restatements of tests/train_ref.py (run in
float64 on the GPU where the case is large): ragged last tiles, NCHW tiles that cross images, ok masks that change
inside a tile, 1-128 classes and 1-48 keypoints on both sides of the 48 KB shared-memory limits, every gamma branch,
every gradient input, the first loss call of a fresh process, and int64 ids that int32 cannot hold.  The inputs and the
bound functions are in tests/train_edge_cases.py; tests/test_train_edges_host.py checks that each bound rejects the
mutants of tests/train_ref.py.

Bounds (u = 2^-24; first-order error terms, then doubled for the second-order ones; CUDA's documented maximum errors
without fast math: expf 2 ulp, logf 1 ulp, powf 4 ulp, and 1 ulp <= 2u relative):
  * focal row.  The max is exact.  Each exp argument z_j - mx is rounded (u |z_j - mx|) and expf adds 4u relative;
    since e^-d d <= 1/e, the C terms carry at most (0.37 C + 4) u relative to their sum, which is >= 1.  The
    sequential float32 sum of C terms adds (C - 1) u.  logf adds 2u L (L = log sum <= a = |logpt|), and the two
    subtractions of logpt = (z_t - mx) - L add u (|z_t - mx| + a) <= 2u a.  So eps(logpt) <= u (4a + 1.4C + 3).
    pt = expf(logpt) is then within eps + 4u, and x = 1 - pt within eps + 5u.  The row is f a with f = x^gamma;
    a gamma x^(gamma-1) <= gamma (1 + a) for every gamma >= 0 (x >= a / (1 + a)), and powf adds 8u f.  So
    |err(row)| <= u (1 + gamma)(1 + a)(4a + 2C + 16) + 9u row.
  * focal loss.  A block sums its 128 rows in a 5-level warp tree and a 4-term sum (8 roundings); blocks are summed
    in float64, cast to float32 (u) and divided by float32(M) (2u, M = 2^24 + 3 is not a float32 integer).  So
    |err| <= 2 [sum_rows u (1 + gamma)(1 + a)(4a + 2C + 16) + 12u sum_rows row] / M (M = 1 for the sum).
  * focal gradient.  dz_j = S f (delta_jt - p_j) with S = g / M.  |delta_jt - p_j| <= x, and x df <= gamma dx + 8u, so
    the f term adds S u gamma (4a + 1.4C + 8) + 8u S; p_j = expf((z_j - mx) - lse) adds u (1.4C + 8 + 4a) S; S, the
    product and the fma add 6u |dz_j|.  |err| <= 2 S u (1 + gamma)(4a + 2C + 16) + 8u |dz_j|.
  * OF loss[b,k] = S / den.  A block's partial is a chain of at most 3 terms per thread (np * 3 <= 384 values on 128
    threads, ragged or not), each |pred - targ| rounded once, a 5-level warp tree and a 4-term block sum: 11 roundings
    on sum w |diff|.  Tiles are added in float64, cast to float32 (u); den = float32(count + 1e-3) equals the
    reference's; the division adds u.  |err| <= 2 (11u S / den + 3u |loss|).
  * OF gradient = (g / den) w sgn(diff), signs exact; g = w_term g_loss + g_parts[term] (+ g_kp) is at most 3
    roundings, the division one: |err| <= 6u |ref| when the g's do not cancel (every g here is >= 0).
  * parts[1], parts[2] and the weighted loss are sequential float32 sums of b K values: a 2 n u sum |value| term on
    top of the values' own bounds.
"""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import train_edge_cases as E
import train_ref as R
from pvn3d_b200 import train_utils as T
from pvn3d_b200._lib import Pvn3dError

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))


def _d(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _check(got, want, bound, what):
    bad = E.exceeds(got, want, bound)
    n = int(bad.sum())
    if n:
        i = int(torch.nonzero(bad.reshape(-1))[0])
        g, w = torch.as_tensor(got).double().reshape(-1)[i], torch.as_tensor(want).double().reshape(-1)[i]
        b = torch.as_tensor(bound, dtype=torch.float64).expand_as(torch.as_tensor(want)).reshape(-1)[i]
        raise AssertionError(f"{what}: {n} values out of bound; first at flat {i}: got {float(g)!r} want "
                             f"{float(w)!r} bound {float(b)!r}")


def _focal(dev, z, t, gamma, mean, what):
    x = _d(z, dev).requires_grad_(True)
    tt = _d(t, dev)
    loss = T.FocalLoss(gamma=gamma, size_average=mean)(x, tt)
    loss.backward()
    rows = R.nchw_rows(_d(z, dev))
    rl, rg = R.focal_t(rows, tt.reshape(-1), gamma, mean=mean)
    lb, gb = E.focal_bounds(rows, tt.reshape(-1), gamma, rg, mean=mean)
    _check(loss.detach(), rl, lb, f"{what} loss")
    _check(R.nchw_rows(x.grad), rg, gb, f"{what} grad")


@pytest.mark.parametrize("c", E.FOCAL_C)
def test_focal_rows(cuda_dev, c):
    for m in E.FOCAL_M:
        z, t = E.focal_rows(m, c, seed=m + 1000 * c)
        for gamma in E.GAMMAS:
            for mean in (True, False):
                _focal(cuda_dev, z, t, gamma, mean, f"[{m},{c}] gamma={gamma} mean={mean}")


def test_focal_nchw_tiles_across_images(cuda_dev):
    for i, shape in enumerate(E.NCHW_SHAPES):
        z, t = E.nchw_case(shape, seed=i)
        for mean in (True, False):
            _focal(cuda_dev, z, t, E.GAMMAS[i % len(E.GAMMAS)], mean, f"{shape} mean={mean}")


def test_focal_large_m(cuda_dev):
    g = torch.Generator(device=cuda_dev).manual_seed(7)
    z = torch.randn(E.LARGE_M, 2, device=cuda_dev, generator=g) * 3
    t = torch.randint(0, 2, (E.LARGE_M,), device=cuda_dev, generator=g)
    for gamma in (2.0, 1.5):
        x = z.clone().requires_grad_(True)
        loss = T.FocalLoss(gamma=gamma)(x, t)
        loss.backward()
        rl, rg = R.focal_t(z, t, gamma)
        lb, gb = E.focal_bounds(z, t, gamma, rg)
        _check(loss.detach(), rl, lb, f"M=2^24+3 gamma={gamma} loss")
        _check(x.grad, rg, gb, f"M=2^24+3 gamma={gamma} grad")
        del x, rg, gb


def _of(dev, pred, targ, lab, g, what):
    p = _d(pred, dev).requires_grad_(True)
    tg, lb_ = _d(targ, dev), _d(lab, dev)
    loss = T.OFLoss()(p, tg, lb_)
    (loss * _d(g, dev)).sum().backward()
    rl, rg = R.of_t(_d(pred, dev), tg, lb_, g=_d(g, dev))
    lb, gb = E.of_bounds(_d(pred, dev), tg, lb_, rl, rg)
    _check(loss.detach(), rl, lb, f"{what} loss")
    _check(p.grad, rg, gb, f"{what} grad")
    return loss.detach(), p.grad


@pytest.mark.parametrize("k", E.OF_K)
def test_of_ragged_tiles(cuda_dev, k):
    for b in E.OF_B:
        for n in E.OF_N:
            pred, targ, lab = E.of_case(b, n, k, seed=n + 7 * k + b)
            g = np.random.default_rng(n).uniform(0.5, 2, (b, k)).astype(np.float32)
            loss, grad = _of(cuda_dev, pred, targ, lab, g, f"b={b} n={n} K={k}")
            if b > 1:     # frame 0 has no labelled point: loss and gradient exactly 0
                assert float(loss[0].abs().max()) == 0 and float(grad[0].abs().max()) == 0


def test_of_float_labels_and_nonfinite_predictions(cuda_dev):
    pred, targ, lab = E.of_nonfinite_case(seed=3)
    g = np.ones((2, 4), np.float32)
    loss, grad = _of(cuda_dev, pred, targ, lab, g, "NaN / inf at unlabelled points, float labels")
    # 0 * |NaN| and 0 * |inf| are NaN in lib/loss.py too: the poisoned (frame, keypoint) terms are NaN, nothing else
    nan = torch.isnan(loss).cpu().numpy()
    assert nan[0, :3].all() and not nan[0, 3] and not nan[1].any()
    # ... but the gradient is finite: torch.abs's backward takes sign(NaN) = 0
    assert bool(torch.isfinite(grad).all()) and float(grad[0, 0, 0].abs().max()) == 0
    # the 1e-8 cut: label 1e-9 weighs nothing, 2e-8 weighs one point
    assert float(grad[0, 3, 1].abs().max()) == 0 and float(grad[0, 3, 2].abs().max()) > 0


@pytest.mark.parametrize("c", E.PVN_C)
def test_pvn3d_loss_ok_mask_weights_and_every_gradient_input(cuda_dev, c):
    ok = torch.tensor(E.PVN_OK, dtype=torch.uint8, device=cuda_dev)
    crit = T.PVN3DLoss(weights=E.PVN_WEIGHTS, gamma=E.PVN_GAMMA)
    for k in E.PVN_K:
        kp, seg, ctr, kt, ct, lab = (_d(a, cuda_dev) for a in E.pvn3d_case(E.PVN_B, E.PVN_N, c, k, seed=c + k))
        for name, (a, v) in E.PVN_GRADS.items():
            what = f"C={c} K={k} backward through {name}"
            ins = [t.clone().requires_grad_(True) for t in (kp, seg, ctr)]
            loss, parts, acc = crit(ins[0], ins[1], ins[2], kt, ct, lab, ok)
            (a * loss + (parts * torch.tensor(v, device=cuda_dev)).sum()).backward()
            ref = R.pvn3d_loss_t(kp, seg, ctr, kt, ct, lab, ok, E.PVN_WEIGHTS, E.PVN_GAMMA, g_loss=a, g_parts=v)
            gs = [a * w + vv for w, vv in zip(E.PVN_WEIGHTS, v)]
            mask = ok.bool().repeat_interleave(E.PVN_N)
            z, t = seg.reshape(-1, c), lab.reshape(-1)
            flb, fgb = E.focal_bounds(z, t, E.PVN_GAMMA, ref["d_seg"].reshape(-1, c), row_mask=mask, g=gs[0])
            kl, kg = R.of_t(kp, kt, lab)
            cl, cg = R.of_t(ctr, ct, lab)
            klb, kgb = E.of_bounds(kp, kt, lab, kl, ref["d_kp"])
            clb, cgb = E.of_bounds(ctr, ct, lab, cl, ref["d_ctr"])
            pb = [flb, E.sum_bound(kl, klb), E.sum_bound(cl, clb)]
            _check(parts, ref["parts"], torch.tensor(pb, dtype=torch.float64), f"{what}: parts")
            wp = [w * float(p) for w, p in zip(E.PVN_WEIGHTS, ref["parts"])]
            lb = sum(w * b for w, b in zip(E.PVN_WEIGHTS, pb)) + 10 * E.U * sum(abs(x) for x in wp)
            _check(loss.detach(), ref["loss"], lb, f"{what}: loss")
            _check(acc, ref["acc"], 2 * E.U, f"{what}: acc")
            _check(ins[1].grad.reshape(-1, c), ref["d_seg"].reshape(-1, c), fgb, f"{what}: d_seg")
            _check(ins[0].grad, ref["d_kp"], kgb, f"{what}: d_kp")
            _check(ins[2].grad, ref["d_ctr"], cgb, f"{what}: d_ctr")
            # the rows of ok = 0 frames, and a term whose g is 0, get exactly 0
            assert float(ins[1].grad[[1, 4]].abs().max()) == 0, what
            for grad, gw in ((ins[1].grad, gs[0]), (ins[0].grad, gs[1]), (ins[2].grad, gs[2])):
                if gw == 0:
                    assert float(grad.abs().max()) == 0, what


_FRESH = r"""
import json, sys
import numpy as np
import torch
sys.path[:0] = [{root!r}, {tests!r}]
import train_edge_cases as E
from pvn3d_b200 import train_utils as T
kind, size, out = sys.argv[1], int(sys.argv[2]), sys.argv[3]
dev = torch.device("cuda:0")
try:
    if kind == "C":          # the first loss call of this process: FocalLoss with C classes, forward and backward
        z, t = E.focal_rows(3 * E.TILE + 5, size, seed=size)
        x = torch.from_numpy(z).to(dev).requires_grad_(True)
        loss = T.FocalLoss(gamma=2)(x, torch.from_numpy(t).to(dev))
    else:                    # ... or OFLoss with K keypoints
        pred, targ, lab = E.of_case(2, 3 * E.TILE + 5, size, seed=size)
        x = torch.from_numpy(pred).to(dev).requires_grad_(True)
        loss = T.OFLoss()(x, torch.from_numpy(targ).to(dev), torch.from_numpy(lab).to(dev))
    loss.sum().backward()
    np.savez(out, loss=loss.detach().cpu().numpy(), grad=x.grad.cpu().numpy())
    print(json.dumps({{"ok": True}}))
except Exception as e:
    print(json.dumps({{"ok": False, "error": repr(e)}}))
"""


def test_first_loss_call_of_a_fresh_process(cuda_dev):
    """The shared-memory opt-in is latched per process and device, so in the pytest process an earlier call with a
    larger footprint would hide a launch that fails without it: each size runs as a process's first loss call."""
    script = _FRESH.format(root=ROOT, tests=TESTS)
    sizes = [("C", c) for c in E.FRESH_C] + [("K", k) for k in E.FRESH_K]
    flags = ["-s"] if sys.flags.no_user_site else []
    results = {}
    with tempfile.TemporaryDirectory() as tmp:
        procs = {}
        try:
            for kind, size in sizes:
                out = os.path.join(tmp, f"{kind}{size}.npz")
                procs[(kind, size)] = (subprocess.Popen([sys.executable, *flags, "-c", script, kind, str(size), out],
                                                        stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                                                        cwd=ROOT), out)
            for key, (p, out) in procs.items():
                so, se = p.communicate(timeout=180)
                line = so.strip().splitlines()[-1] if so.strip() else "{}"
                results[key] = (json.loads(line) if line.startswith("{") else {"ok": False}, out, se[-2000:])
        finally:
            for p, _ in procs.values():
                if p.poll() is None:
                    p.kill()
                    p.wait()
        failed = {f"{k}={s}": r[0].get("error", r[2]) for (k, s), r in results.items() if not r[0].get("ok")}
        assert not failed, f"first loss call failed: {failed}"
        for (kind, size), (_, out, _) in results.items():
            got = np.load(out)
            dev = cuda_dev
            if kind == "C":
                z, t = E.focal_rows(3 * E.TILE + 5, size, seed=size)
                rl, rg = R.focal_t(_d(z, dev), _d(t, dev), 2.0)
                lb, gb = E.focal_bounds(_d(z, dev), _d(t, dev), 2.0, rg)
            else:
                pred, targ, lab = E.of_case(2, 3 * E.TILE + 5, size, seed=size)
                rl, rg = R.of_t(_d(pred, dev), _d(targ, dev), _d(lab, dev))
                lb, gb = E.of_bounds(_d(pred, dev), _d(targ, dev), _d(lab, dev), rl, rg)
            _check(_d(got["loss"], dev), rl, lb, f"fresh process {kind}={size} loss")
            _check(_d(got["grad"], dev), rg, gb, f"fresh process {kind}={size} grad")


def _check_targets(got, want, what):
    for g, w, name in zip(got, want, ("kp_targ_ofst", "ctr_targ_ofst", "kp3ds", "ctr3ds")):
        g = g.cpu().numpy()
        assert g.shape == w.shape, (what, name)
        ia, ib = g.view(np.int32).astype(np.int64), w.view(np.int32).astype(np.int64)
        ia = np.where(ia < 0, -(ia & 0x7fffffff), ia)
        ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
        assert np.abs(ia - ib).max(initial=0) <= 1, f"{what} {name}"   # float32 of a float64 value: 1 ulp


def _targets(dev, case, what):
    pcld, labels, ids, rts, kp, ctr = case
    tt = T.TrainTargets(kp_table=kp, ctr_table=ctr, device=dev)
    got = tt.compute(_d(pcld, dev), _d(labels, dev), _d(ids, dev), _d(rts, dev))
    _check_targets(got, R.targets_ref(pcld, labels, ids, rts, kp, ctr), what)
    return got


def test_targets_int64_ids_beyond_int32(cuda_dev):
    case = E.targets_case(4, 600, 22, 8, 22, seed=1, wide=True)
    got = _targets(cuda_dev, case, "int64 ids")
    labels, ids = case[1], case[2]
    wide = np.isin(labels, E.WIDE_IDS)
    assert wide.sum() >= 12 and np.abs(got[0].cpu().numpy()[wide]).max() == 0
    assert float(got[2][0, 0].abs().max()) == 0 and float(got[2][:, -1].abs().max()) == 0   # wide slot ids: empty


def test_targets_ragged_blocks_k_and_full_shared_memory(cuda_dev):
    for n in E.TGT_N:
        for k in E.TGT_K:
            _targets(cuda_dev, E.targets_case(3, n, 1, k, 22, seed=n + k), f"n={n} K={k} S=1")
    s, k, n_cls = E.TGT_FULL
    assert E.tgt_smem(s, k, n_cls) == E.TGT_MAX_SMEM
    _targets(cuda_dev, E.targets_case(2, E.TGT_THREADS + 3, s, k, n_cls, seed=5), "shared memory exactly full")
    case = E.targets_case(1, 4, s, k, n_cls + 1, seed=6)
    with pytest.raises(Pvn3dError, match="unsupported"):   # one class more: 4 B over, refused before any launch
        T.TrainTargets(kp_table=case[4], ctr_table=case[5], device=cuda_dev).compute(
            *(_d(a, cuda_dev) for a in case[:4]))


def test_targets_one_point_per_frame(cuda_dev):
    case = E.targets_case(E.TGT_MANY_FRAMES, 1, 2, 1, 5, seed=9)
    _targets(cuda_dev, case, f"{E.TGT_MANY_FRAMES} frames of one point")


def test_same_bits_and_no_host_sync(cuda_dev):
    kp, seg, ctr, kt, ct, lab = (_d(a, cuda_dev) for a in E.pvn3d_case(E.PVN_B, E.PVN_N, 96, 32, seed=1))
    ok = torch.tensor(E.PVN_OK, dtype=torch.uint8, device=cuda_dev)
    crit = T.PVN3DLoss(weights=E.PVN_WEIGHTS, gamma=E.PVN_GAMMA)

    def run():
        ins = [t.clone().requires_grad_(True) for t in (kp, seg, ctr)]
        loss, parts, acc = crit(ins[0], ins[1], ins[2], kt, ct, lab, ok)
        (loss + parts.sum()).backward()
        return [loss.detach(), parts.detach(), acc] + [t.grad for t in ins]

    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        first = run()
        second = run()
        z = seg.reshape(-1, 96).clone().requires_grad_(True)
        T.FocalLoss(gamma=0.5)(z, lab.reshape(-1)).backward()
        p = kp.clone().requires_grad_(True)
        T.OFLoss()(p, kt, lab).sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert all(torch.equal(a, b) for a, b in zip(first, second))
    z2 = seg.reshape(-1, 96).clone().requires_grad_(True)
    T.FocalLoss(gamma=0.5)(z2, lab.reshape(-1)).backward()
    p2 = kp.clone().requires_grad_(True)
    T.OFLoss()(p2, kt, lab).sum().backward()
    assert torch.equal(z.grad, z2.grad) and torch.equal(p.grad, p2.grad)
