"""CPU checks of the fused-forward references of tests/pn2_forward_ref.py, on 2 frames x 4096 points with the seeded
model and the oracle's index ops:

  * a float32 emulation of the factored forward (the factor table, TF32 operands in fp32 matmuls, V as the fp32 fma
    chain, tf32(relu(U[idx] - V)), layers 2 and 3, the max-pool, the FP interpolation's fma chain and the rounding each
    SA level stores) lies inside every launch's float64 bound;
  * every mutant lies outside its bound on the same data, at the launches R.MUTANTS names;
  * without the TF32 rounding, the float64 twin of the module graph reproduces the float32 module graph (oracle ops,
    oracle/ext_cpu.py) to float32 noise.
"""
import copy
import types

import numpy as np
import pytest
import torch

import geo_ref as G
import pn2_forward_ref as R
from oracle import ext_cpu, pn2
from pvn3d_b200 import synth, testing
from pvn3d_b200.mlp import tf32_round
from pvn3d_b200.pointnet2 import SA_SPEC

B, N = 2, 4096


@pytest.fixture(scope="module")
def case():
    cloud = synth.stack(synth.make_batch("ycb", B, n_points=N, config_id=41))["cld_rgb_nrm"]
    l_xyz, ball, nn = [np.ascontiguousarray(cloud[..., :3])], [], {}
    for npoint, radii, nsamples, _ in SA_SPEC:
        l_xyz.append(G.gather_rows(l_xyz[-1], pn2.furthest_point_sampling(l_xyz[-1], npoint)))
        ball.append([torch.from_numpy(pn2.ball_query(l_xyz[-1], l_xyz[-2], float(np.float32(r)), ns))
                     for r, ns in zip(radii, nsamples)])
    for i in range(4):
        d2, idx = pn2.three_nn(l_xyz[i], l_xyz[i + 1])
        nn[i] = (torch.from_numpy(idx), torch.from_numpy(G.weights_ref(d2)))
    plan = types.SimpleNamespace(l_xyz=[torch.from_numpy(x) for x in l_xyz], ball=ball, nn=nn)
    model = testing.seeded_pointnet2msg(0, 1)
    W = R.model_weights(model, "cpu")
    cloud = torch.from_numpy(cloud)
    return cloud, plan, model, W, emulate(cloud, plan, W)


def _fma(a, b, c):
    """fmaf: the float32 product is exact in float64, one rounding of the sum (to float64, then float32: a double
    rounding that can differ from fmaf in the last bit, far inside every bound)"""
    return (a.double() * b.double() + c.double()).float()


def _interp(p, idx, w, m):
    """the kernels' three-point interpolation fma(p2, w2, fma(p0, w0, p1 * w1)) in float32"""
    b = idx.size(0)
    rows = (torch.arange(b)[:, None, None] * m + idx.long()).reshape(-1, 3)
    w = w.reshape(-1, 3, 1)
    q = p[rows]
    return _fma(q[:, 2], w[:, 2], _fma(q[:, 0], w[:, 0], q[:, 1] * w[:, 1]))


def emulate(cloud, plan, W):
    """the factored forward of FusedPointnet2MSG.features in float32 on the CPU -> the namespace recording() fills"""
    b, n0, width = cloud.shape
    cap = types.SimpleNamespace(u=[], v=[], level=[], fp={})
    f = cloud[..., 3:]
    for li, (_, _, nsamples, _) in enumerate(SA_SPEC):
        x, c = plan.l_xyz[li], plan.l_xyz[li + 1]
        n, m = x.size(1), c.size(1)
        hi = tf32_round(x)
        table = torch.cat([tf32_round(f), hi, tf32_round(x - hi)], -1).reshape(b * n, -1)
        cf = c.reshape(-1, 3)
        us, vs, outs = [], [], []
        for w, ns in zip(W.sa[li], nsamples):
            u = table @ tf32_round(torch.cat([w.wf, w.wx, w.wx], 1)).t()
            v = _fma(cf[:, 2:3], w.wx[:, 2], _fma(cf[:, 1:2], w.wx[:, 1], cf[:, :1] * w.wx[:, 0])) - w.b1
            idx = plan.ball[li][len(us)].long()
            rows_u = (torch.arange(b)[:, None, None] * n + idx).reshape(-1)
            a = tf32_round(torch.relu(u[rows_u] - v.repeat_interleave(ns, 0)))
            h = tf32_round(torch.relu(a @ w.w2.t() + w.b2))
            outs.append(torch.relu(h @ w.w3.t() + w.b3).view(-1, ns, w.w3.size(0)).amax(1))
            us.append(u)
            vs.append(v)
        level = torch.cat(outs, 1)
        cap.level.append(tf32_round(level) if li < 3 else level)
        cap.u.append(us)
        cap.v.append(vs)
        f = cap.level[-1].view(b, m, -1)
    for i in (3, 2, 1):
        known = cap.level[3] if i == 3 else cap.fp[i + 1]
        p = W.fp[i]
        a = torch.cat([tf32_round(_interp(known, *plan.nn[i], plan.l_xyz[i + 1].size(1))), cap.level[i - 1]], 1)
        h = tf32_round(torch.relu(a @ p.w1.t() + p.b1))
        cap.fp[i] = torch.relu(h @ p.w2.t() + p.b2)
    cap.p = tf32_round(cap.fp[1]) @ W.fp1.wk.t()
    x = cloud[..., :3]
    hi = tf32_round(x)
    table0 = torch.cat([tf32_round(cloud[..., 3:]), hi, tf32_round(x - hi)], -1).reshape(b * n0, -1)
    s = table0[:, :width - 3] @ W.fp1.ws.t() + W.fp1.bs
    a = tf32_round(torch.relu(_interp(cap.p, *plan.nn[0], plan.l_xyz[1].size(1)) + s))
    cap.out = torch.relu(a @ W.fp1.w2.t() + W.fp1.b2).view(b, n0, -1).transpose(1, 2).contiguous()
    return cap


def test_emulation_inside_every_bound(case):
    cloud, plan, _, W, cap = case
    for name, _, build in R.launches():
        worst = R.check_launch(build, cap, plan, cloud, W, 1, name)
        print(f"{name}: worst |got - ref| / bound {worst:.3g}")


@pytest.mark.parametrize("mutant", list(R.MUTANTS))
def test_every_mutant_outside_its_bound(case, mutant):
    """each required rejection is asserted inside try_mutant; the rest are reported (see R.MUTANTS for why)"""
    cloud, plan, _, W, cap = case
    R.try_mutant(mutant, cap, plan, cloud, W, 1)


def _cpu_ops():
    def three_nn(unknown, known):
        d2, idx = ext_cpu.three_nn(unknown, known)
        return torch.sqrt(d2), idx

    return {"furthest_point_sample": ext_cpu.furthest_point_sampling,
            "ball_query": lambda radius, nsample, xyz, new_xyz: ext_cpu.ball_query(new_xyz, xyz, radius, nsample),
            "three_nn": three_nn}


def test_f64_twin_reproduces_the_fp32_module_graph(case):
    """the twin the GPU test measures the engine against: with no TF32 rounding it is the float32 module graph's
    computation in float64 -- the same neighbours, the same dataflow -- so the two differ by float32 noise only"""
    cloud, plan, model, _, _ = case
    log = {k: [] for k in R.DISCRETE}
    ops = dict(R.recorder(log, _cpu_ops()), gather_operation=R.t_gather, grouping_operation=R.t_group,
               three_interpolate=R.t_interp)
    out32 = R.module_forward(copy.deepcopy(model), cloud, ops)
    assert [len(log[k]) for k in R.DISCRETE] == [4, 8, 4]
    for li in range(4):                                  # the recorded choices are the plan's
        for s in range(2):
            assert torch.equal(log["ball_query"][2 * li + s], plan.ball[li][s])
        assert torch.equal(log["three_nn"][li][1], plan.nn[3 - li][0])
    out64 = R.module_forward(copy.deepcopy(model).double(), cloud.double(), R.twin(log, True))
    err = R.frame_errors(out32, out64)
    print("fp32 module graph vs float64 twin, per frame (mean, p99.9):", err.tolist())
    assert (err[:, 0] <= 2e-6).all() and (err[:, 1] <= 2e-5).all(), err
