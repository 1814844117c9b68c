"""One training step of the staged reference PVN3D (as test_deterministic_gpu.py builds it: B = 2, 480 x 640,
N = 12288) under torch.autocast, in a subprocess:

  (a) the step completes under bf16 and under fp16 autocast (before the 16-bit entry points, SA2's group_points
      raised "points must be a float tensor");
  (b) the pvn3d_*_16 entry points were reached, counted per entry point;
  (c) the loss and every parameter gradient are finite, and the loss is within LOSS_GAP of the float32 step on the
      same inputs and parameters;
  (d) with compat's deterministic patch and torch.use_deterministic_algorithms(True), two bf16 steps give the same
      bits in every gradient, and so do two fp16 steps;
  (e) the step also runs in a fresh thread inside torch.amp.autocast("cuda", enabled=True) -- what an
      nn.DataParallel replica runs -- and reaches the fp16 entry points there, whatever dtype the main thread set.
"""
import json
import math
import os
import subprocess
import sys
import textwrap

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# |loss16 - loss32| / |loss32| on the step below, measured on an H100 80GB HBM3 (700 W): 5.7e-6 (bf16) and 1.4e-4
# (fp16).  The bounds leave a margin of about 18x (bf16) and 7x (fp16).
LOSS_GAP = {"bf16": 1e-4, "fp16": 1e-3}

STEP = textwrap.dedent("""
    import json, sys, threading
    import torch
    sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
    from helpers import load_reference_python
    from pvn3d_b200 import _ext, compat, deterministic
    ref = load_reference_python()
    assert ref is not None
    compat.install(patch_deterministic=True)
    counts = {{}}
    def counting(real):
        def call(fn, dev, *args):
            if fn.endswith("_16"):
                key = fn + (":f16" if args[0] == 1 else ":bf16")
                counts[key] = counts.get(key, 0) + 1
            return real(fn, dev, *args)
        return call
    _ext.call = counting(_ext.call)
    deterministic.call = counting(deterministic.call)
    import lib.pvn3d as P
    from lib.loss import FocalLoss, OFLoss
    from lib.pspnet import Modified_PSPNet
    P.modified_psp_models["resnet34"] = lambda: Modified_PSPNet(sizes=(1, 2, 3, 6), psp_size=512,
                                                                deep_features_size=256, backend="resnet34",
                                                                pretrained=False)
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    model = P.PVN3D(num_classes=22, pcld_input_channels=6, pcld_use_xyz=True, num_kps=8, num_points=12288).to(dev)
    model.train()
    crit, crit_of = FocalLoss(gamma=2), OFLoss()
    b, n = 2, 12288
    gen = torch.Generator().manual_seed(1)
    rgb = torch.rand((b, 3, 480, 640), generator=gen).to(dev)
    cld = torch.randn((b, n, 9), generator=gen).to(dev) * 0.1
    choose = torch.stack([torch.randperm(480 * 640, generator=gen)[:n] for _ in range(b)])[:, None].to(dev)
    labels = torch.randint(0, 22, (b, n), generator=gen).to(dev)
    kp_targ = torch.randn((b, n, 8, 3), generator=gen).to(dev) * 0.05
    ctr_targ = torch.randn((b, n, 1, 3), generator=gen).to(dev) * 0.05
    DT = {{"fp32": None, "bf16": torch.bfloat16, "fp16": torch.float16}}

    def forward():
        pred_kp_of, pred_rgbd_seg, pred_ctr_of = model(cld, rgb, choose)
        return (crit(pred_rgbd_seg.view(labels.numel(), -1), labels.view(-1)).sum() * 2.0
                + crit_of(pred_kp_of, kp_targ, labels).sum() + crit_of(pred_ctr_of, ctr_targ, labels).sum())

    def run(mode):
        torch.manual_seed(2)
        model.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=DT[mode], enabled=DT[mode] is not None):
            loss = forward()
        loss.backward()
        torch.cuda.synchronize()
        return loss.detach().float().clone(), {{k: p.grad.detach().clone() for k, p in model.named_parameters()
                                                if p.grad is not None}}

    def finite(grads):
        return all(bool(torch.isfinite(g).all()) for g in grads.values())

    res = {{}}
    for mode in ("fp32", "bf16", "fp16"):
        counts.clear()
        try:
            loss, grads = run(mode)
        except RuntimeError as e:
            res[mode] = {{"raised": str(e)[:400]}}
            continue
        res[mode] = {{"loss": float(loss), "params": len(grads), "finite": finite(grads), "calls": dict(counts)}}
    torch.use_deterministic_algorithms(True)
    for mode in ("bf16", "fp16"):
        counts.clear()
        try:
            (l1, g1), (l2, g2) = run(mode), run(mode)
        except RuntimeError as e:
            res["det_" + mode] = {{"raised": str(e)[:400]}}
            continue
        same = [k for k in g1 if torch.equal(g1[k].view(torch.int8), g2[k].view(torch.int8))]
        res["det_" + mode] = {{"loss": [float(l1), float(l2)], "params": len(g1), "bit_equal": len(same),
                               "differ": [k for k in g1 if k not in same][:10], "finite": finite(g1),
                               "calls": dict(counts)}}
    torch.use_deterministic_algorithms(False)

    # a DataParallel replica: a fresh thread, autocast enabled without a dtype
    torch.set_autocast_dtype("cuda", torch.bfloat16)
    counts.clear()
    out = {{}}
    def replica():
        try:
            torch.manual_seed(2)
            model.zero_grad(set_to_none=True)
            with torch.amp.autocast("cuda", enabled=True):
                out["dtype"] = str(torch.get_autocast_dtype("cuda"))
                loss = forward()
            loss.backward()
            torch.cuda.synchronize()
            out["loss"] = float(loss)
            out["finite"] = finite({{k: p.grad for k, p in model.named_parameters() if p.grad is not None}})
        except RuntimeError as e:
            out["raised"] = str(e)[:400]
    t = threading.Thread(target=replica)
    t.start()
    t.join()
    out["calls"] = dict(counts)
    res["thread"] = out
    print(json.dumps(res))
""")


@pytest.fixture(scope="module")
def step_results(cuda_dev):
    if not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "py", "lib")):
        pytest.skip("the reference Python is not staged under oracle/_ref/py")
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    code = STEP.format(root=ROOT, tests=os.path.join(ROOT, "tests"))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT, timeout=1800)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    print(json.dumps(res, indent=1))
    return res


ENTRY = ["pvn3d_group_points_16", "pvn3d_three_interpolate_16"]


@pytest.mark.parametrize("mode", ["bf16", "fp16"])
def test_autocast_step_completes_and_reaches_the_16_bit_ops(step_results, mode):
    res = step_results[mode]
    assert "raised" not in res, res
    code = ":f16" if mode == "fp16" else ":bf16"
    for fn in ENTRY + ["pvn3d_group_points_grad_16", "pvn3d_three_interpolate_grad_16"]:
        assert res["calls"].get(fn + code, 0) > 0, (fn, res["calls"])
    assert not any(k.endswith(":f16" if mode == "bf16" else ":bf16") for k in res["calls"]), res["calls"]


@pytest.mark.parametrize("mode", ["bf16", "fp16"])
def test_autocast_loss_and_gradients_are_finite_and_near_float32(step_results, mode):
    ref, res = step_results["fp32"], step_results[mode]
    assert "raised" not in ref and "raised" not in res, (ref, res)
    assert ref["calls"] == {}, ref["calls"]                   # float32 runs only the float32 entry points
    assert ref["finite"] and res["finite"] and math.isfinite(res["loss"]), res
    assert res["params"] == ref["params"] > 100
    gap = abs(res["loss"] - ref["loss"]) / abs(ref["loss"])
    print(f"{mode}: loss {res['loss']:.6g} vs float32 {ref['loss']:.6g}, relative gap {gap:.3g}")
    assert gap <= LOSS_GAP[mode], (gap, res["loss"], ref["loss"])


@pytest.mark.parametrize("mode", ["bf16", "fp16"])
def test_deterministic_autocast_steps_repeat_bit_for_bit(step_results, mode):
    res = step_results["det_" + mode]
    assert "raised" not in res, res
    assert res["loss"][0] == res["loss"][1] and res["finite"], res
    assert res["params"] > 100 and res["bit_equal"] == res["params"], res
    code = ":f16" if mode == "fp16" else ":bf16"
    for fn in ("pvn3d_group_points_grad_ordered_16", "pvn3d_three_interpolate_grad_ordered_16",
               "pvn3d_upsample_bilinear2d_backward_16", "pvn3d_adaptive_avg_pool2d_backward_16"):
        assert res["calls"].get(fn + code, 0) > 0, (fn, res["calls"])


def test_replica_thread_autocast_runs_fp16(step_results):
    res = step_results["thread"]
    assert "raised" not in res, res
    assert res["dtype"] == "torch.float16" and res["finite"], res
    for fn in ENTRY + ["pvn3d_group_points_grad_16", "pvn3d_three_interpolate_grad_16"]:
        assert res["calls"].get(fn + ":f16", 0) > 0, (fn, res["calls"])
