"""Whole PVN3D training steps against a float64 twin: every parameter gradient of the staged reference model's step
(resnet34 Modified_PSPNet without pretrained weights, 22 classes, 8 keypoints, N = 12288, B = 2, 480 x 640), with this
package's PointNet++ ops, its deterministic backward, its fused loss and its 16-bit paths, each measured against a
pure-torch twin of the same precision.

The inputs come from the package's own training input path (train_utils.train_batch on two synthetic scenes: real
balls, FPS over a scene, foreground labels and offset targets).  model_fn's loss is 2 focal + sum kp OF + sum ctr OF.
Every Dropout2d has p = 0, cuDNN is deterministic without benchmarking and TF32 is off, so the arms differ only in the
operations this package supplies; one state_dict is reloaded before each arm (train-mode BatchNorm updates its running
statistics).  All arms run in one subprocess, because the deterministic arms need CUBLAS_WORKSPACE_CONFIG before CUDA
starts:

  * "float64": the model in float64 on torch replays of the six module-level ops of lib.pointnet2_utils (the FPS /
    ball / 3-NN choices recorded from the first package arm, tests/train_step_ref.py), the reference's lib.loss in
    float64, deterministic mode off;
  * "torch fp32", "torch bf16", "torch fp16": the same replays in float32, and under autocast with the kernels'
    16-bit contract (compute in float32, round each output once), reference loss -- the error baseline of each
    precision;
  * the package arms, fp32 / bf16 / fp16 x atomic / deterministic (compat's patch_deterministic with
    torch.use_deterministic_algorithms) x the reference loss / the fused loss (compat's patch_loss):
    pvn3d_b200._ext under the unmodified reference model.

fp16 steps scale the loss by FP16_SCALE as GradScaler does; gradients are divided by it in float64 and must be finite.

Checks: the package arms make the FPS / ball / 3-NN choices the twins replay; each loss is within twice its twin's
error of the float64 loss + 1e-7 (relative); each of the 268 parameter gradients has (mean, p99.9) of
|g - g64| / mean|g64| within twice its twin's + a floor (FLOOR); a gradient that is exactly zero in float64 is exactly
zero in every arm.  The fp32 twin itself is held to float64 in absolute terms (TWIN32_SANITY), so a wrong twin cannot
quietly widen every bound.

Two kinds of gradient are sums that cancel far below their terms, and for them |g - g64| is divided by sum |term| of
each element (taken from hooks on the float64 step) instead of by mean |g64|:
  * the bias of a convolution that feeds a train-mode BatchNorm (PSPUpsample's): zero in exact arithmetic, so its
    float64 value is rounding noise;
  * each PSPUpsample PReLU slope, one element summing dL/dy * min(x, 0) over a whole feature map: its fp32 value has a
    relative error near 2e-3 (H100, this step), so its statistic is one sample of rounding noise, and correct fp32
    arms landed up to 2.2x the fp32 twin's error.
For these sums the statistic is one or a few samples of rounding noise, and the twins' own noise changes from run to
run (with deterministic mode off, torch's upsample / pooling / gather backward add with atomics).  So their floor,
CANCEL_FLOOR, is one unit roundoff of the arm's precision in sum |term| units: the one rounding of each term to a
16-bit dtype alone moves such a sum by up to u16 sum |term| in any correct arm, whatever its twin drew.

The check must bite: four wrong wirings, injected by wrapping the package's Python entry points in the subprocess,
each fail the fp32 gradient check on the same data (MUTANTS).
"""
import copy
import gc
import json
import math
import os
import subprocess
import sys
import time

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
B, N = 2, 12288
FP16_SCALE = 2.0 ** 12
N_PARAMS = 268                    # parameters of the reference PVN3D that the loss reaches
# Floors in units of mean |g64|.  On an H100 80GB HBM3 every 16-bit gradient outside the cancelling sums below was
# within twice its autocast twin's error with no floor at all (worst error / (2 x twin error) 0.74 fp16, 0.62 - 0.70
# bf16, over three runs of the module); those arms take the fp32 floor, which matters only where a twin's error is
# near zero.
FLOOR = {"fp32": 1e-6, "bf16": 1e-6, "fp16": 1e-6}
# Floors of the cancelling sums, in units of sum |term|: the unit roundoff of each precision (u = 2^-8 for bfloat16's 8
# significant bits, 2^-11 for float16's 11); fp32 keeps 1e-6 (17 u32).
# Measured on an H100 80GB HBM3, three runs of the module: the 16-bit PReLU slopes' errors were 4e-4 - 1.3e-3 (bf16,
# at most 0.34 u) and 2e-5 - 3.4e-4 (fp16, at most 0.7 u), the conv biases' below 6e-5; the fp32 ones at most 0.81 of
# their bound, with the same value in all three runs.
CANCEL_FLOOR = {"fp32": 1e-6, "bf16": 2.0 ** -8, "fp16": 2.0 ** -11}
# the fp32 twin against float64, in absolute terms: the relative loss error, the median over the parameters of the mean
# error, and the largest mean error.  Measured (H100, three runs): 1.1e-7, 9.3e-3 and 3.4e-2 -- train-mode BatchNorm
# over the whole network and max-pool choices that flip between float32 and float64 move most gradients by about 1 %.
# The bounds are 5-9x those: loose, there to stop a wrong twin (an O(1) error) from widening every bound.
TWIN32_SANITY = {"loss": 1e-6, "median": 0.05, "max": 0.2}
PRECISIONS = ("fp32", "bf16", "fp16")
ARMS = [f"{p} {mode} {loss}" for p in PRECISIONS for mode in ("atomic", "deterministic") for loss in ("ref", "fused")]
MUTANTS = {
    "ordered group grad, first slot of each run dropped": "fp32 deterministic ref",
    "PSP upsample backward, align_corners flipped at up_3": "fp32 deterministic ref",
    "interpolate grad, weights of points j and j+1 swapped": "fp32 atomic ref",
    "fused loss backward scaled by 1 + 2^-8": "fp32 atomic fused",
}


def _floor(arm, param, res):
    """the floor of one parameter's bound in an arm (a mutant arm: its fp32 arm's)"""
    p = MUTANTS[arm[len("mutant: "):]].split()[0] if arm.startswith("mutant: ") else arm.split()[0]
    return CANCEL_FLOOR[p] if param in res["cancelled"] else FLOOR[p]


# ---- the subprocess --------------------------------------------------------------------------------------------------
def _subprocess():
    import torch

    import train_ref
    import train_step_ref as R
    from helpers import load_reference_python

    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    ref = load_reference_python()
    assert ref is not None
    import lib.loss as L
    import lib.pvn3d as P
    from lib.pspnet import Modified_PSPNet
    from pvn3d_b200 import _ext, compat, deterministic
    from pvn3d_b200 import train_utils as T
    from pvn3d_b200.frame_input import FrameInputBuilder

    # lib/loss.py's own losses, made before patch_loss rebinds the names (FocalLoss.__init__ calls
    # super(FocalLoss, self), which looks the name up again), then the drop-ins patch_loss installs
    ref_loss = (L.FocalLoss(gamma=2), L.OFLoss())
    compat.install(patch_deterministic=True, patch_loss=True)
    fused_loss = (L.FocalLoss(gamma=2), L.OFLoss())
    assert isinstance(fused_loss[0], T.FocalLoss) and isinstance(fused_loss[1], T.OFLoss)
    P.modified_psp_models["resnet34"] = lambda: Modified_PSPNet(sizes=(1, 2, 3, 6), psp_size=512,
                                                                deep_features_size=256, backend="resnet34",
                                                                pretrained=False)
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    model = P.PVN3D(num_classes=22, pcld_input_channels=6, pcld_use_xyz=True, num_kps=8, num_points=N).to(dev).train()
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout2d):
            m.p = 0.0
    state = copy.deepcopy(model.state_dict())
    model64 = copy.deepcopy(model).double()

    # gradients that are sums cancelling far below their terms, and sum |term| of each, from hooks on the float64 step:
    # the bias of a conv feeding a train-mode BatchNorm (sum over n, h, w of dL/dy per channel: zero in exact
    # arithmetic) and each PReLU slope (sum of dL/dy * min(x, 0))
    sums, hooks = {}, []
    mods64 = dict(model64.named_modules())
    for name, mod in model.named_modules():
        if isinstance(mod, torch.nn.Sequential):
            kids = list(mod.named_children())
            for (a, ma), (b, mb) in zip(kids, kids[1:]):
                if isinstance(ma, torch.nn.modules.conv._ConvNd) and ma.bias is not None and \
                        isinstance(mb, torch.nn.modules.batchnorm._BatchNorm):
                    key = f"{name}.{a}.bias"
                    hooks.append(mods64[f"{name}.{a}"].register_full_backward_hook(
                        lambda m, gi, go, key=key: sums.__setitem__(key, go[0].abs().sum((0, 2, 3)))))
        if isinstance(mod, torch.nn.PReLU):
            key, x_in = f"{name}.weight", {}
            hooks.append(mods64[name].register_forward_hook(lambda m, i, o, x_in=x_in: x_in.__setitem__(0, i[0])))
            hooks.append(mods64[name].register_full_backward_hook(
                lambda m, gi, go, key=key, x_in=x_in: sums.__setitem__(
                    key, (go[0] * x_in.pop(0).clamp(max=0)).abs().sum().reshape(1))))
    del mods64, x_in

    arrays = train_ref.raw_frames(B)
    depth, K, cs, rgb, label, ids, rts = (torch.from_numpy(a).to(dev) for a in arrays)
    builder = FrameInputBuilder(B, N, device=dev)
    batch = T.train_batch(builder, T.TrainTargets(device=dev), depth, K, cs, rgb, label, ids, rts, seed=11)
    rgb_o, _, cld, choose, kp_t, ctr_t, _, _, labels, _, _, ok = (t.clone() for t in batch)
    assert ok.tolist() == [1] * B
    fg = int((labels > 0).sum())
    x32 = dict(cld=cld, rgb=rgb_o, choose=choose, kp=kp_t, ctr=ctr_t, labels=labels)
    x64 = {k: v.double() if v.is_floating_point() else v for k, v in x32.items()}

    pu = ref.pn2_utils
    discrete = {k: getattr(pu, k) for k in R.DISCRETE}
    amp = {"fp32": None, "bf16": torch.bfloat16, "fp16": torch.float16}

    def step(mdl, x, losses, prec, det=False, ops=()):
        scale = FP16_SCALE if prec == "fp16" else 1.0
        mdl.load_state_dict(state)
        mdl.zero_grad(set_to_none=True)
        torch.manual_seed(2)
        crit, crit_of = losses
        ops = dict(ops)
        saved = {k: getattr(pu, k) for k in ops}
        t0 = time.time()
        try:
            for k, fn in ops.items():
                setattr(pu, k, fn)
            torch.use_deterministic_algorithms(det)
            with torch.autocast("cuda", dtype=amp.get(prec), enabled=amp.get(prec) is not None):
                kp, seg, ctr = mdl(x["cld"], x["rgb"], x["choose"])
                loss = (crit(seg.view(x["labels"].numel(), -1), x["labels"].view(-1)).sum() * 2.0
                        + crit_of(kp, x["kp"], x["labels"]).sum() + crit_of(ctr, x["ctr"], x["labels"]).sum())
            (loss * scale).backward()
            torch.cuda.synchronize()
        finally:
            torch.use_deterministic_algorithms(False)
            for k, fn in saved.items():
                setattr(pu, k, fn)
        grads = {k: p.grad.detach().double() / scale for k, p in mdl.named_parameters() if p.grad is not None}
        return float(loss.detach().double()), grads, time.time() - t0

    res = {"arms": {}, "fg_points": fg}
    log = {k: [] for k in R.DISCRETE}
    g64 = scales = None

    def record(name, loss, grads, secs, choices=None):
        finite = all(bool(torch.isfinite(g).all()) for g in grads.values())
        out = {"loss": loss, "finite": finite, "params": len(grads), "seconds": round(secs, 3), "err": {},
               "nonzero_where_f64_zero": []}
        if choices is not None:
            out["choices_equal"] = choices
        if g64 is not None:
            assert set(grads) == set(g64), name
            for k, g in grads.items():
                if float(g64[k].abs().max()) == 0.0:
                    if float(g.abs().max()) != 0.0:
                        out["nonzero_where_f64_zero"].append(k)
                    continue
                out["err"][k] = R.err(g, g64[k], scales[k])
        res["arms"][name] = out
        print(f"[{name}] loss {loss:.9g} finite {finite} {secs:.2f} s", file=sys.stderr, flush=True)

    def measured(run):
        """run() -> (its result, GiB allocated before it, peak GiB allocated while it ran)"""
        gc.collect()
        torch.cuda.synchronize(dev)
        torch.cuda.empty_cache()
        held = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        out = run()
        return out, held / 2 ** 30, torch.cuda.max_memory_allocated(dev) / 2 ** 30

    def same_choices(new):
        return all(len(new[k]) == len(log[k]) for k in R.DISCRETE) and all(
            all(torch.equal(u, v) for u, v in zip(a if isinstance(a, (list, tuple)) else [a],
                                                   b if isinstance(b, (list, tuple)) else [b]))
            for k in R.DISCRETE for a, b in zip(new[k], log[k]))

    def package(prec, det, loss_kind, name=None):
        mine = {k: [] for k in R.DISCRETE}
        loss, grads, secs = step(model, x32, fused_loss if loss_kind == "fused" else ref_loss, prec, det,
                                 R.recorder(mine, discrete))
        mode = "deterministic" if det else "atomic"
        record(name or f"{prec} {mode} {loss_kind}", loss, grads, secs, same_choices(mine))

    # a first fp32 package step records the choices every twin replays (and the fp32 arm checks it makes them again)
    step(model, x32, ref_loss, "fp32", False, R.recorder(log, discrete))
    assert [len(log[k]) for k in R.DISCRETE] == [4, 8, 4], {k: len(v) for k, v in log.items()}
    model.zero_grad(set_to_none=True)
    (loss64, g64, secs64), *res["float64_gib"] = measured(
        lambda: step(model64, x64, ref_loss, "float64", False, R.twin(log, True)))
    for h in hooks:
        h.remove()
    del model64, hooks
    scales = {k: sums.get(k, float(g64[k].abs().mean())) for k in g64}
    res["cancelled"] = sorted(sums)
    record("float64", loss64, g64, secs64)
    for prec in PRECISIONS:
        record(f"torch {prec}", *step(model, x32, ref_loss, prec, False, R.twin(log, False)))
    for arm in ARMS:
        prec, mode, loss_kind = arm.split()
        if arm == "fp32 atomic ref":
            _, *res["fp32_gib"] = measured(lambda: package(prec, mode == "deterministic", loss_kind))
        else:
            package(prec, mode == "deterministic", loss_kind)

    # ---- mutants: wrong wirings of the package's Python entry points
    def mutant(name, install, uninstall):
        prec, mode, loss_kind = MUTANTS[name].split()
        install()
        try:
            package(prec, mode == "deterministic", loss_kind, "mutant: " + name)
        finally:
            uninstall()

    def swap_attr(obj, attr, new):
        old = getattr(obj, attr)
        return (lambda: setattr(obj, attr, new(old))), (lambda: setattr(obj, attr, old))

    mutant("ordered group grad, first slot of each run dropped", *swap_attr(
        _ext, "group_points_grad",
        lambda real: lambda g, idx, n: real(R.drop_first_of_run(g, idx).contiguous(), idx, n)))
    seen = {"align": 0}

    def flip_align(real):
        def call(fn, dev_, *args):
            if fn.startswith("pvn3d_upsample_bilinear2d_backward"):
                k = 1 if fn.endswith("_16") else 0
                if args[k + 6] == 1:                     # align_corners=True: the PSPUpsample stages, up_3 first
                    seen["align"] += 1
                    if seen["align"] == 1:
                        args = args[:k + 6] + (0,) + args[k + 7:]
            return real(fn, dev_, *args)
        return call
    mutant("PSP upsample backward, align_corners flipped at up_3", *swap_attr(deterministic, "call", flip_align))
    res["align_calls"] = seen["align"]
    mutant("interpolate grad, weights of points j and j+1 swapped", *swap_attr(
        _ext, "three_interpolate_grad", lambda real: lambda g, idx, w, m: real(g, idx, R.swap_pairs(w), m)))
    real_bw = T._TrainLoss.backward

    def scaled_bw(ctx, *g):
        return tuple(None if t is None else t * R.LOSS_SCALE_MUTANT for t in real_bw(ctx, *g))
    mutant("fused loss backward scaled by 1 + 2^-8",
           lambda: setattr(T._TrainLoss, "backward", staticmethod(scaled_bw)),
           lambda: setattr(T._TrainLoss, "backward", staticmethod(real_bw)))
    res["gpu"] = torch.cuda.get_device_name(dev)
    print(json.dumps(res))


# ---- the checks ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def step_results(cuda_dev):
    if not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "py", "lib")):
        pytest.skip("the reference Python is not staged under oracle/_ref/py")
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    t0 = time.time()
    r = subprocess.run([sys.executable, os.path.abspath(__file__)], capture_output=True, text=True, env=env, cwd=ROOT,
                       timeout=3000)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    print(r.stderr[-3000:])
    print(f"subprocess wall time {time.time() - t0:.1f} s on {res['gpu']}; {res['fg_points']} foreground points; "
          f"cancelling sums {res['cancelled']}")
    for what, key in (("float64 step", "float64_gib"), ("fp32 atomic step", "fp32_gib")):
        held, peak = res[key]
        print(f"{what}: peak allocated {peak:.2f} GiB, of which {held:.2f} GiB was held before the step (models, "
              f"inputs, recorded choices; before the fp32 step also the float64 gradients) and {peak - held:.2f} GiB "
              f"is the step's own")
    return res


def _arm(res, name):
    a = res["arms"][name]
    assert a["finite"], name                               # fp16: no inf or NaN after the loss scale
    assert a["params"] == N_PARAMS, (name, a["params"])
    return a


def _twin_of(arm):
    """the twin an arm is measured against (a mutant arm: its fp32 arm's)"""
    if arm.startswith("mutant: "):
        arm = MUTANTS[arm[len("mutant: "):]]
    return "torch " + arm.split()[0]


def _outside(res, arm):
    """{parameter: (arm error, twin error)} of the gradients outside their bound"""
    a, t = res["arms"][arm], res["arms"][_twin_of(arm)]
    return {k: (e, t["err"][k]) for k, e in a["err"].items()
            if not all(x <= 2 * y + _floor(arm, k, res) for x, y in zip(e, t["err"][k]))}


def test_twins_are_complete(step_results):
    for name in ("float64",) + tuple("torch " + p for p in PRECISIONS):
        _arm(step_results, name)
    assert step_results["cancelled"] == [f"cnn.model.up_{i}.conv.{j}.{p}" for i in (1, 2, 3)
                                         for j, p in ((1, "bias"), (3, "weight"))]
    assert step_results["fg_points"] > 1000


def test_fp32_twin_is_near_float64(step_results):
    """a wrong fp32 twin would widen every fp32 bound: hold it to float64 in absolute terms"""
    l64 = step_results["arms"]["float64"]["loss"]
    t = step_results["arms"]["torch fp32"]
    means = sorted(e[0] for e in t["err"].values())
    loss_err, median = abs(t["loss"] - l64) / abs(l64), means[len(means) // 2]
    print(f"torch fp32 against float64: loss {loss_err:.3g}, mean error median {median:.3g}, largest {means[-1]:.3g}")
    assert loss_err <= TWIN32_SANITY["loss"] and median <= TWIN32_SANITY["median"] and \
        means[-1] <= TWIN32_SANITY["max"], (loss_err, median, means[-1])


@pytest.mark.parametrize("arm", ARMS)
def test_discrete_choices_equal_the_replayed_ones(step_results, arm):
    assert _arm(step_results, arm)["choices_equal"], arm


@pytest.mark.parametrize("arm", ARMS)
def test_loss_within_twice_the_twin_error(step_results, arm):
    l64 = step_results["arms"]["float64"]["loss"]
    la = _arm(step_results, arm)["loss"]
    lt = step_results["arms"][_twin_of(arm)]["loss"]
    ea, et = abs(la - l64) / abs(l64), abs(lt - l64) / abs(l64)
    print(f"{arm}: loss {la:.9g}, float64 {l64:.9g}: relative error {ea:.3g}, {_twin_of(arm)} {et:.3g}")
    assert ea <= 2 * et + 1e-7, (arm, ea, et)


@pytest.mark.parametrize("arm", ARMS)
def test_parameter_gradients_within_twice_the_twin_error(step_results, arm):
    a = _arm(step_results, arm)
    assert not a["nonzero_where_f64_zero"], a["nonzero_where_f64_zero"]
    bad = _outside(step_results, arm)
    assert not bad, (arm, dict(list(bad.items())[:8]))


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_mutants_fail_the_gradient_check(step_results, mutant):
    name = "mutant: " + mutant
    a = _arm(step_results, name)
    assert a["choices_equal"]
    bad = _outside(step_results, name)
    worst = sorted(bad.items(), key=lambda kv: -max(x / max(2 * y, 1e-300) for x, y in zip(*kv[1])))[:3]
    print(f"mutant {mutant!r}: {len(bad)} of {len(a['err'])} gradients outside the bound, e.g. {worst}")
    assert bad, mutant
    if mutant.startswith("PSP"):
        assert step_results["align_calls"] == 3


def test_zz_report_worst_ratios(step_results):
    """prints, per arm and module family, the largest (error - floor) / (2 x twin error) over both statistics, the
    three largest parameters, and the ratios of the cancelling sums"""
    import train_step_ref as R
    res = step_results
    for arm in ARMS + ["mutant: " + m for m in MUTANTS]:
        a, twin = res["arms"][arm], res["arms"][_twin_of(arm)]
        ratios = {k: R.ratio(e, twin["err"][k], _floor(arm, k, res)) for k, e in a["err"].items()}
        worst = {}
        for k, r in ratios.items():
            worst[R.family(k)] = max(worst.get(R.family(k), -math.inf), r)
        plain = {k: r for k, r in ratios.items() if k not in res["cancelled"]}
        top = sorted(plain, key=plain.get)[-3:][::-1]
        print(f"F64RATIO {arm}: " + ", ".join(f"{f} {v:.3g}" for f, v in sorted(worst.items())) + "; largest outside "
              "the cancelling sums at " + ", ".join(f"{k} {plain[k]:.3g} {a['err'][k]}" for k in top))
        print(f"CANCELRATIO {arm}: " + ", ".join(f"{k} {ratios[k]:.3g} {a['err'][k]} twin {twin['err'][k]}"
                                                 for k in res["cancelled"]))


if __name__ == "__main__":
    sys.path.insert(0, ROOT)                  # the script's own directory, tests/, is already first
    _subprocess()
