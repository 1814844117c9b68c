"""References of the fused Pointnet2MSG forward (`FusedPointnet2MSG.features`) built from the model's dataflow
(`Pointnet2MSG.forward`, pvn3d_b200/pointnet2.py) -- test infrastructure, importable without a GPU.

  * `recording(engine)`: records the output of every launch of one `features()` call -- U and V of each (level, scale),
    each SA level table, each FP2-FP4 output, P and the network output -- by wrapping the module globals `mlp_dense`,
    `sa_centre_term`, `mlp_fp2`, `mlp_fp_fact2` of pvn3d_b200.mlp and the per-scale fused callables of `engine.sa`.
    The engine's code is not changed.
  * float64 references of every launch with the element-wise bounds of tests/f64_bounds.py.  A reference is built from
    the model's own layers (`fold_conv_bn` + `tf32_round`), the plan's coordinates, ball rows and 3-NN rows / weights
    (held bit-exact to the oracle by tests/test_geometry_bench_gpu.py) and the captured OUTPUTS of earlier launches --
    never from the arguments the engine passed to a launch, so a wrong skip pointer or column offset in `features()`
    cannot be copied into its own reference.
  * wrong references ("mutants", `MUTANTS`) that each check must reject on the same data.
  * the float64 twin of the module graph: `recorder` / `twin` replay the FPS / ball-query / 3-NN choices of a recorded
    run with pure-torch gathers, and `tf32_operands` rounds every conv's operands to TF32 (the cuDNN-TF32 precision
    class, emulated exactly).

Every function works on whatever device its tensors live on; the references of one launch are built for a slice of
frames at a time (`check_launch`), so their peak memory stays bounded at the benchmark's batches.
"""
from __future__ import annotations

import contextlib
import io
import math
import types

import numpy as np
import torch

import f64_bounds as fb
import geo_ref as G
from pvn3d_b200 import mlp, pointnet2
from pvn3d_b200.mlp import fold_conv_bn, tf32_round
from pvn3d_b200.pointnet2 import SA_SPEC

SPLIT = 2.0 ** -21      # |hi + lo - x| of the factor table's coordinate split, relative to |x|


# ---- the launch recorder ---------------------------------------------------------------------------------------------
_WRAPPED = ("mlp_dense", "sa_centre_term", "mlp_fp2", "mlp_fp_fact2")


@contextlib.contextmanager
def recording(engine):
    """-> a namespace filled, when the block ends, with the outputs of the `features()` call made inside it:
    u[li][s], v[li][s] (U and V of SA level li, scale s), level[li] (the SA level table [B*npoint, C]), fp[i] (FP2-FP4
    for i = 1..3, [B*n_i, C]), p (FP1's P = W_k . known) and out ([B,128,N])"""
    events = []
    orig = {name: getattr(mlp, name) for name in _WRAPPED}

    def wrap(name, fn):
        def rec(*a, **k):
            out = fn(*a, **k)
            events.append((name, out))
            return out
        return rec

    sa = engine.sa
    cap = types.SimpleNamespace()
    try:
        for name in _WRAPPED:
            setattr(mlp, name, wrap(name, orig[name]))
        engine.sa = [[(l2, l3, wrap("sa", fused)) for l2, l3, fused in level] for level in sa]
        yield cap
    finally:
        engine.sa = sa
        for name in _WRAPPED:
            setattr(mlp, name, orig[name])
    names = [e[0] for e in events]
    want = ["mlp_dense", "sa_centre_term", "sa"] * 8 + ["mlp_fp2"] * 3 + ["mlp_dense", "mlp_fp_fact2"]
    assert names == want, names
    outs = [e[1] for e in events]
    cap.u = [[outs[3 * (2 * li + s)] for s in range(2)] for li in range(4)]
    cap.v = [[outs[3 * (2 * li + s) + 1] for s in range(2)] for li in range(4)]
    cap.level = [outs[3 * (2 * li + 1) + 2] for li in range(4)]
    assert all(outs[3 * (2 * li) + 2] is not None and outs[3 * (2 * li) + 2].data_ptr() == cap.level[li].data_ptr()
               for li in range(4))
    cap.fp = {3 - k: outs[24 + k] for k in range(3)}
    cap.p, cap.out = outs[27], outs[28]


# ---- the model's weights ---------------------------------------------------------------------------------------------
def model_weights(model, dev):
    """every layer of the model folded (`fold_conv_bn`) and TF32-rounded, unpadded, in the model's column order:
    sa[li][s] (wf, wx = the first layer's feature / xyz columns, b1, w2, b2, w3, b3), fp[i] for i = 1..3 (w1 over
    [interpolated | skip], b1, w2, b2), fp1 (wk, ws = the first layer's known / skip columns, bs, w2, b2)"""
    def fold(layer):
        w, b = fold_conv_bn(layer)
        return tf32_round(w.to(dev)), b.to(dev)

    sa = []
    for mod in model.SA_modules:
        scales = []
        for seq in mod.mlps:
            w1, b1 = fold(seq[0])                                       # columns [xyz(3) | features]
            w2, b2 = fold(seq[1])
            w3, b3 = fold(seq[2])
            scales.append(types.SimpleNamespace(wf=w1[:, 3:].contiguous(), wx=w1[:, :3].contiguous(), b1=b1, w2=w2,
                                                b2=b2, w3=w3, b3=b3))
        sa.append(scales)
    fp = {}
    for i in (1, 2, 3):
        seq = model.FP_modules[i].mlp
        (w1, b1), (w2, b2) = fold(seq[0]), fold(seq[1])
        fp[i] = types.SimpleNamespace(w1=w1, b1=b1, w2=w2, b2=b2)
    seq = model.FP_modules[0].mlp
    (w1, b1), (w2, b2) = fold(seq[0]), fold(seq[1])
    c_skip = model.SA_modules[0].mlps[0][0].conv.weight.size(1) - 3     # FP1's skip is the cloud's descriptors
    ck = w1.size(1) - c_skip
    fp1 = types.SimpleNamespace(wk=w1[:, :ck].contiguous(), ws=w1[:, ck:].contiguous(), bs=b1, w2=w2, b2=b2)
    return types.SimpleNamespace(sa=sa, fp=fp, fp1=fp1)


def _padded(w, shape):
    out = torch.zeros(shape, dtype=w.dtype, device=w.device)
    out[tuple(slice(0, s) for s in w.shape)] = w
    return out


def packed_like_model(engine, W):
    """-> the names of the engine's packed tensors that are NOT bit-equal to the model's folded, TF32-rounded, zero-padded
    layers (first SA layers packed [W_f | W_x | W_x] with a zero bias, Wx and b1 of the centre term, FP1 split into
    W_k and [W_s | 0])"""
    bad = []

    def same(name, got, want):
        if not (got.shape == want.shape and torch.equal(got.view(torch.int32), want.view(torch.int32))):
            bad.append(name)

    def layer(name, pl, w, b):
        same(name + ".w", pl.w, _padded(w, pl.w.shape))
        same(name + ".bias", pl.bias, _padded(b, pl.bias.shape))

    for li in range(4):
        for s in range(2):
            w = W.sa[li][s]
            first, wx, b1 = engine.sa_fact[li][s]
            l2, l3, _ = engine.sa[li][s]
            layer(f"SA{li + 1}.{s}.first", first, torch.cat([w.wf, w.wx, w.wx], 1), torch.zeros_like(w.b1))
            same(f"SA{li + 1}.{s}.wx", wx, _padded(w.wx, wx.shape))
            same(f"SA{li + 1}.{s}.b1", b1, _padded(w.b1, b1.shape))
            layer(f"SA{li + 1}.{s}.l2", l2, w.w2, w.b2)
            layer(f"SA{li + 1}.{s}.l3", l3, w.w3, w.b3)
    for i in (1, 2, 3):
        l1, l2 = engine.fp[i]
        layer(f"FP{i + 1}.l1", l1, W.fp[i].w1, W.fp[i].b1)
        layer(f"FP{i + 1}.l2", l2, W.fp[i].w2, W.fp[i].b2)
    lk, ls, l2 = engine.fp1
    layer("FP1.k", lk, W.fp1.wk, torch.zeros_like(W.fp1.bs))
    layer("FP1.s", ls, W.fp1.ws, W.fp1.bs)
    layer("FP1.l2", l2, W.fp1.w2, W.fp1.b2)
    return bad


# ---- per-launch references -------------------------------------------------------------------------------------------
#: mutant -> (the launch families it is applied to, the launches whose check must reject it).  The others are tried and
#: reported: with the seeded model the features are O(100) and vary little between points and frames (a per-point
#: standard deviation of about a tenth of the mean), so a TF32 ulp of an activation, carried through a layer's |W|^T,
#: is as large as what some mutants move:
#:   * "no lo" at SA2-SA4: the bound of U holds ACC |f| . |W_f|^T over 64-512 feature columns, which dwarfs the
#:     2^-12 |W_x| . |x| of a lost lo (the factor table itself is held bit-exact, lo included, by
#:     tests/test_pn2_edges_gpu.py);
#:   * "roll nn" / "roll skip" at FP4 and "swap nn weights" at FP2-FP4: neighbouring points' SA4 / FP features differ
#:     by little more than the interpolated operand's TF32 ulp carried through 1024 + 512 columns;
#:   * "no bs": FP1's b_s (mean |b_s| 0.13) is about one TF32 ulp of its pre-activation (|P + S| ~ 200), so no
#:     element-wise bound of the output can see it dropped; the engine's b_s is held bit-equal to the model's by
#:     `packed_like_model`, and the kernel's use of it by tests/test_mlp_fused_f64_gpu.py.
MUTANTS = {
    "roll ball": (("sa1", "sa"), ("SA",)),                       # frame b's reference from frame b-1's ball rows
    "roll nn": (("fp", "fp1"), ("FP3", "FP2", "FP1 output")),    # ... from frame b-1's 3-NN rows and weights
    "roll skip": (("fp",), ("FP3", "FP2")),                      # ... from frame b-1's skip table
    "swap scales": (("sa",), ("SA",)),                           # the two scales' column slices of a table swapped
    "no lo": (("sa1",), ("SA1",)),                               # the coordinates' hi half only (mut_table_no_lo)
    "swap nn weights": (("fp", "fp1"), ("FP1 output",)),         # 3-NN weights 1 <-> 2
    "no bs": (("fp1",), ()),                                     # FP1 without its bias b_s
}


def mutant_cases(mutant):
    """(name, reference builder, whether its check must reject the mutant) of every launch the mutant applies to"""
    families, required = MUTANTS[mutant]
    return [(name, build, name.startswith(required)) for name, family, build in launches() if family in families]


def try_mutant(mutant, cap, plan, cloud, W, chunk):
    """-> {launch: None if its check rejected the mutant, else the worst ratio it kept}; asserts every required
    rejection"""
    res = {}
    for name, build, required in mutant_cases(mutant):
        try:
            res[name] = check_launch(build, cap, plan, cloud, W, chunk, name, mutant)
        except AssertionError as e:
            if "outside the bound" not in str(e):
                raise
            res[name] = None
        print(f"mutant {mutant!r} at {name}: " + ("rejected" if res[name] is None else
                                                  f"inside the bound (worst ratio {res[name]:.3g})"))
        assert res[name] is None or not required, (mutant, name, res[name])
    return res


def _rows(x, n, frames):
    """[B*n, C] row table -> [len(frames), n, C]"""
    return x.view(-1, n, x.size(-1))[frames]


def _frames(fr, b, roll):
    """the frames a reference reads for the frames of slice fr (b - 1 for b under a rolled-plan mutant)"""
    f = torch.arange(fr.start, fr.stop)
    return (f - 1) % b if roll else f


def _offsets(k, m, dev):
    return torch.arange(k, device=dev)[:, None, None] * m


def sa_layer1(cap, plan, cloud, W, li, s, fr, mut=None):
    """SA level li, scale s, layer 1 before its ReLU, every grouped row of the frames fr.  Engine: fl32(U[idx] - V) from
    the captured U and V.  Reference: the unfactored W_f . tf32(f_j) + W_x . (x_j - c) + b1 in float64, f_j from the
    captured table of level li - 1 (level 0: the cloud's descriptors), x_j from l_xyz[li], c from l_xyz[li + 1], rows
    from the plan's ball table.  Bound: ACC |[f|hi|lo]| . |[W_f|W_x|W_x]|^T for U, centre_term_f64's for V, 2^-21
    |W_x| . |x| for the hi / lo split and one fp32 subtraction."""
    b = plan.l_xyz[0].size(0)
    x32, c32 = plan.l_xyz[li], plan.l_xyz[li + 1]
    n, m = x32.size(1), c32.size(1)
    dev = x32.device
    w = W.sa[li][s]
    wf, wx, b1 = w.wf.double(), w.wx.double(), w.b1.double()
    n1 = wf.size(0)
    rows = plan.ball[li][s][_frames(fr, b, False)].long()                            # the engine's rows
    idx = plan.ball[li][s][_frames(fr, b, mut == "roll ball")].long()                # the reference's
    k, _, ns = idx.shape
    fi = torch.arange(k, device=dev)[:, None, None]
    x32 = x32[fr]
    tab = G.factor_table_ref(x32.reshape(-1, 3).cpu().numpy(), None, 0, 6)         # [hi | lo] of every point
    split = torch.from_numpy(tab).to(dev).double().view(k, n, 6)
    x = x32.double()
    if mut == "no lo":
        t = torch.from_numpy(G.mut_table_no_lo(tab, 0)).to(dev).double().view(k, n, 6)
        x = t[..., :3] + t[..., 3:]
    f = cloud[fr][..., 3:] if li == 0 else _rows(cap.level[li - 1], n, fr)
    f = fb.tf32(f)
    c = c32[fr].double()
    uf = f @ wf.t()                                                                    # per point
    eu = fb.ACC * (f.abs() @ wf.abs().t() + split.abs() @ torch.cat([wx, wx], 1).abs().t())
    eu = eu + SPLIT * (x32.double().abs() @ wx.abs().t())
    _, ev = G.centre_term_f64(c.reshape(-1, 3).cpu().numpy(), wx.cpu().numpy(), b1.cpu().numpy())
    ev = torch.from_numpy(ev).to(dev).view(k, m, 1, n1)
    ref = uf[fi, idx] + (x[fi, idx] - c[:, :, None]) @ wx.t() + b1
    bound = eu[fi, idx] + ev
    bound = bound + fb.F32 * (ref.abs() + bound)
    got = _rows(cap.u[li][s], n, fr)[fi, rows] - _rows(cap.v[li][s], m, fr)[:, :, None]
    return got.reshape(-1, n1), ref.reshape(-1, n1), bound.reshape(-1, n1)


def sa_scale_out(cap, plan, W, li, s, fr, mut=None):
    """SA level li, scale s, layers 2 and 3 + max-pool: fb.sa_scale on the captured U and V with the model's W2 / W3
    (TF32-rounded output for SA1-SA3) against the scale's columns of the captured level table, the column offset summed
    from the model's layer widths"""
    b = plan.l_xyz[0].size(0)
    n, m = plan.l_xyz[li].size(1), plan.l_xyz[li + 1].size(1)
    w = W.sa[li][s]
    idx = plan.ball[li][s][_frames(fr, b, mut == "roll ball")].long()
    k, _, ns = idx.shape
    dev = idx.device
    rows_u = ((fr.start + torch.arange(k, device=dev))[:, None, None] * n + idx).reshape(-1)
    rows_v = torch.arange(fr.start * m, (fr.start + k) * m, device=dev).repeat_interleave(ns)
    ref, bound = fb.sa_scale(cap.u[li][s], cap.v[li][s], rows_u, rows_v, w.w2, w.b2, w.w3, w.b3, ns, round_out=li < 3)
    widths = [sc.w3.size(0) for sc in W.sa[li]]
    col = sum(widths[s + 1:]) if mut == "swap scales" else sum(widths[:s])
    got = _rows(cap.level[li], m, fr)[..., col:col + widths[s]]
    return got.reshape(-1, widths[s]), ref, bound


def fp_out(cap, plan, W, i, fr, mut=None):
    """FP module i (FP2-FP4 for i = 1..3): fb.fp_module with the captured table below as the known input (SA4's for
    FP4), the captured SA level i table as the skip input and the plan's 3-NN rows and weights"""
    b = plan.l_xyz[0].size(0)
    n, m = plan.l_xyz[i].size(1), plan.l_xyz[i + 1].size(1)
    p = W.fp[i]
    known = cap.level[3] if i == 3 else cap.fp[i + 1]
    skip = cap.level[i - 1]
    c1 = skip.size(-1)
    nn_idx, nn_w = (t[_frames(fr, b, mut == "roll nn")] for t in plan.nn[i])
    if mut == "swap nn weights":
        nn_w = nn_w[..., [1, 0, 2]]
    k = nn_idx.size(0)
    rows = (_offsets(k, m, nn_idx.device) + nn_idx.long()).reshape(-1, 3)
    sk = skip.view(b, n, c1)[_frames(fr, b, mut == "roll skip")]
    ref, bound = fb.fp_module(_rows(known, m, fr).reshape(-1, known.size(-1)), rows, nn_w.reshape(-1, 3),
                              sk.reshape(-1, c1), c1, p.w1, p.b1, p.w2, p.b2, round_out=False)
    return _rows(cap.fp[i], n, fr).reshape(-1, p.w2.size(0)), ref, bound


def fp1_p(cap, plan, W, fr, mut=None):
    """FP1's P = W_k . tf32(FP2 output), once per level-1 point"""
    m = plan.l_xyz[1].size(1)
    a = fb.tf32(_rows(cap.fp[1], m, fr).reshape(-1, cap.fp[1].size(-1)))
    wk = W.fp1.wk
    ref, bound = fb.dense(a, wk, torch.zeros(wk.size(0), dtype=torch.float64, device=a.device), relu=False)
    return _rows(cap.p, m, fr).reshape(-1, cap.p.size(-1)), ref, bound


def fp1_out(cap, plan, cloud, W, fr, mut=None):
    """the network output: fb.fp1_module on the captured P, the plan's 3-NN rows and weights and the level-0 factor table
    of the cloud (geo_ref.factor_table_ref); compared point-major"""
    b, n, width = cloud.shape
    m = plan.l_xyz[1].size(1)
    c0 = width - 3
    nn_idx, nn_w = (t[_frames(fr, b, mut == "roll nn")] for t in plan.nn[0])
    if mut == "swap nn weights":
        nn_w = nn_w[..., [1, 0, 2]]
    k = nn_idx.size(0)
    dev = nn_idx.device
    rows = (_offsets(k, m, dev) + nn_idx.long()).reshape(-1, 3)
    pts = cloud[fr].reshape(-1, width).cpu().numpy()
    table = torch.from_numpy(G.factor_table_ref(pts[:, :3], pts[:, 3:], c0, c0 + 6)).to(dev)
    ws = _padded(W.fp1.ws, (W.fp1.ws.size(0), c0 + 6))
    bs = torch.zeros_like(W.fp1.bs) if mut == "no bs" else W.fp1.bs
    ref, bound = fb.fp1_module(_rows(cap.p, m, fr).reshape(-1, cap.p.size(-1)), rows, nn_w.reshape(-1, 3), table, ws,
                               bs, W.fp1.w2, W.fp1.b2, round_out=False)
    return cap.out[fr].transpose(1, 2).reshape(-1, cap.out.size(1)), ref, bound


def launches():
    """(name, family, reference builder (cap, plan, cloud, W, fr, mut) -> (got, ref, bound)) of every launch, in the
    order features() runs them"""
    out = []
    for li in range(4):
        for s in range(2):
            out.append((f"SA{li + 1} scale {s} layer 1", "sa1",
                        lambda c, p, x, W, fr, mut, li=li, s=s: sa_layer1(c, p, x, W, li, s, fr, mut)))
            out.append((f"SA{li + 1} scale {s} layers 2-3 + max-pool", "sa",
                        lambda c, p, x, W, fr, mut, li=li, s=s: sa_scale_out(c, p, W, li, s, fr, mut)))
    for i in (3, 2, 1):
        out.append((f"FP{i + 1}", "fp", lambda c, p, x, W, fr, mut, i=i: fp_out(c, p, W, i, fr, mut)))
    out.append(("FP1 P", "p", lambda c, p, x, W, fr, mut: fp1_p(c, p, W, fr, mut)))
    out.append(("FP1 output", "fp1", lambda c, p, x, W, fr, mut: fp1_out(c, p, x, W, fr, mut)))
    return out


def check_launch(build, cap, plan, cloud, W, chunk, what, mut=None):
    """fb.check of one launch over every frame, `chunk` frames per reference; -> the worst |got - ref| / bound (raises
    fb.check's AssertionError, "outside the bound", at the first chunk with an element outside)"""
    b = cloud.size(0)
    worst = 0.0
    for f0 in range(0, b, chunk):
        fr = slice(f0, min(b, f0 + chunk))
        got, ref, bound = build(cap, plan, cloud, W, fr, mut)
        with contextlib.redirect_stdout(io.StringIO()):
            worst = max(worst, fb.check(got, ref, bound, f"{what}, frames {fr.start}..{fr.stop - 1}"))
    return worst


# ---- the module graph's float64 twin ---------------------------------------------------------------------------------
DISCRETE = ("furthest_point_sample", "ball_query", "three_nn")


def t_gather(features, idx):
    b, c = features.shape[:2]
    return features.gather(2, idx.long()[:, None].expand(b, c, idx.size(1)))


def t_group(features, idx):
    b, c = features.shape[:2]
    return features.gather(2, idx.long().reshape(b, 1, -1).expand(b, c, -1)).reshape(b, c, *idx.shape[1:])


def t_interp(features, idx, weight):
    return (t_group(features, idx) * weight[:, None]).sum(-1)


def recorder(log, ops=None):
    """the discrete ops (pointnet2's own, or `ops`), each appending its output to log[name]"""
    orig = ops if ops is not None else {k: getattr(pointnet2, k) for k in DISCRETE}

    def wrap(name):
        def fn(*a):
            out = orig[name](*a)
            log[name].append(out)
            return out
        return fn
    return {k: wrap(k) for k in DISCRETE}


def twin(log, f64):
    """pure-torch ops that replay the recorded FPS / ball-query / 3-NN choices (f64: the 3-NN distances recomputed from
    the float64 coordinates)"""
    its = {k: iter(v) for k, v in log.items()}

    def nn(unknown, known):
        dist, idx = next(its["three_nn"])
        if f64:                                          # the same neighbours, their float64 distances
            b, n = idx.shape[:2]
            k = known.detach().gather(1, idx.long().reshape(b, -1, 1).expand(b, n * 3, 3)).reshape(b, n, 3, 3)
            dist = (unknown.detach()[:, :, None] - k).square().sum(-1).sqrt()
        return dist, idx

    return {"furthest_point_sample": lambda xyz, npoint: next(its["furthest_point_sample"]),
            "ball_query": lambda radius, nsample, xyz, new_xyz: next(its["ball_query"]),
            "three_nn": nn, "gather_operation": t_gather, "grouping_operation": t_group,
            "three_interpolate": t_interp}


def tf32_operands(model):
    """round every conv's weight (now) and input (at every call) to TF32 with fb.tf32: the TF32 precision class of
    cuDNN emulated exactly, independent of the algorithm cuDNN picks.  In place; returns the model."""
    for mod in model.modules():
        if isinstance(mod, torch.nn.Conv2d):
            with torch.no_grad():
                mod.weight.copy_(fb.tf32(mod.weight))
            mod.register_forward_pre_hook(lambda _, a: (fb.tf32(a[0]),))
    return model


@contextlib.contextmanager
def patched(ops):
    """pointnet2's module-level ops replaced by `ops` inside the block"""
    orig = {k: getattr(pointnet2, k) for k in ops}
    try:
        for k, fn in ops.items():
            setattr(pointnet2, k, fn)
        yield
    finally:
        for k, fn in orig.items():
            setattr(pointnet2, k, fn)


def module_forward(model, pc, ops):
    """the module graph's forward on pc with pointnet2's ops replaced by `ops`, detached.  The input requires grad so that
    QueryAndGroup takes the ball_query + grouping_operation path (without autograd it runs the fused kernel, which
    neither replays a recorded choice nor takes float64)."""
    with patched(ops), torch.enable_grad():
        return model(pc.detach().clone().requires_grad_(True)).detach()


def frame_errors(out, ref):
    """per frame: (mean, 99.9th percentile) of |out - ref| / mean |ref|, [B, 2] float64"""
    res = []
    for o, r in zip(out, ref):
        e = ((o.double() - r).abs() / r.abs().mean()).flatten()
        res.append((float(e.mean()), float(e.kthvalue(max(1, math.ceil(0.999 * e.numel()))).values)))
    return np.array(res)
