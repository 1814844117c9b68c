"""The fused Pointnet2MSG forward (`FusedPointnet2MSG.features`, hot path A) at the three shapes bench.py times --
LineMOD 32 x 12288, YCB 16 x 12288 and the stress configuration 8 x 49152, clouds built as bench.Runner builds them --
every frame, launch by launch and end to end, against float64 references built from the model's dataflow
(tests/pn2_forward_ref.py).  The engine is that of `testing.seeded_pointnet2msg(0, 1)`.

  * the engine's packed weights are the model's folded, TF32-rounded layers bit for bit, and recording the launches of
    a `features()` call changes neither its bits nor its launch count;
  * every launch within its float64 bound: the first layer of all 8 SA scales (unfactored, from the captured table of
    the level below), layers 2-3 + max-pool of each scale at its model-derived column offset, FP4-FP2, P and FP1;
  * the checks reject wiring mutants on the same data (a plan rolled by one frame, swapped scale columns, the
    coordinates' hi half only, swapped neighbour weights, FP1 without b_s -- R.MUTANTS names where each must be
    rejected and why the rest cannot be), and an engine re-run of SA1 with the `lo` columns of its factor table zeroed
    fails its layer-1 check;
  * end to end, per frame: the output's error against the float64 twin of the module graph (replaying the engine's own
    FPS / ball / 3-NN choices) is at most 2x that of the same twin with TF32-rounded conv operands, plus 1e-6;
  * batch invariance: each frame's output bits do not depend on the other frames of the batch nor on its place in it.

On an H100 80GB HBM3 at a 700 W power limit the file's 40 tests take 21 s.  The launch checks of one configuration take
0.2-0.8 s and its end-to-end arms 0.5-1.7 s; the references are built four frames at a time, which keeps their peak
memory at a few GB.  Measured there: worst |got - ref| / bound per launch family 0.05 (SA layer 1), 0.53 (SA layers
2-3), 0.006 (FP2-FP4), 0.04 (P), 0.11 (FP1); the engine's per-frame error over the TF32-operand twin's 0.77-1.16.
"""
import copy
import time
import types

import numpy as np
import pytest
import torch

import bench
import pn2_forward_ref as R
from helpers import t
from pvn3d_b200 import _lib, mlp, testing
from test_geometry_bench_gpu import bench_cloud

pytestmark = pytest.mark.gpu

CHUNK = 4        # frames per reference: SA3's grouped rows of 32 frames would take ~4 GB in float64 in one go


@pytest.fixture(scope="module")
def model(cuda_dev):
    return testing.seeded_pointnet2msg(0, 1).to(cuda_dev)


@pytest.fixture(scope="module")
def engine(cuda_dev, model):
    return mlp.FusedPointnet2MSG(model, cuda_dev)


@pytest.fixture(scope="module")
def weights(cuda_dev, model):
    return R.model_weights(model, cuda_dev)


@pytest.fixture(scope="module", params=list(bench.CONFIGS))
def case(request, cuda_dev, engine):
    cloud = t(bench_cloud(request.param), cuda_dev)
    plan = engine.geometry(cloud)
    with R.recording(engine) as cap:
        engine.features(cloud, plan)
    torch.cuda.synchronize()
    return request.param, cloud, plan, cap


def _bits(x):
    return x.contiguous().view(torch.int32)


def test_packed_weights_are_the_models(engine, weights):
    assert R.packed_like_model(engine, weights) == []


def test_recording_changes_no_bit_and_no_launch(case, engine):
    name, cloud, plan, cap = case
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.pvn3d_launch_count()
    plain = engine.features(cloud, plan)
    torch.cuda.synchronize()
    n1 = lib.pvn3d_launch_count()
    with R.recording(engine) as again:
        rec = engine.features(cloud, plan)
    torch.cuda.synchronize()
    n2 = lib.pvn3d_launch_count()
    print(f"[{name}] features(): {n1 - n0} launches plain, {n2 - n1} recorded")
    assert n1 - n0 == n2 - n1 > 0
    assert rec is again.out
    assert torch.equal(_bits(plain), _bits(rec)) and torch.equal(_bits(plain), _bits(cap.out)), name


def test_every_launch_within_f64_bound(case, weights):
    name, cloud, plan, cap = case
    t0 = time.perf_counter()
    fam = {}
    for launch, family, build in R.launches():
        worst = R.check_launch(build, cap, plan, cloud, weights, CHUNK, f"[{name}] {launch}")
        print(f"[{name}] {launch}: worst |got - ref| / bound {worst:.3g}")
        fam[family] = max(fam.get(family, 0.0), worst)
    print(f"[{name}] worst ratio per family {({k: round(v, 3) for k, v in fam.items()})}, "
          f"{time.perf_counter() - t0:.1f} s")


@pytest.mark.parametrize("mutant", list(R.MUTANTS))
def test_checks_reject_wiring_mutants(case, weights, mutant):
    name, cloud, plan, cap = case
    print(f"[{name}]")
    R.try_mutant(mutant, cap, plan, cloud, weights, CHUNK)


@pytest.mark.parametrize("s", [0, 1])
def test_engine_without_lo_fails_the_sa1_layer1_check(case, engine, weights, s):
    """SA1, scale s re-run through the engine's public kernel wrappers: with the factor table as the engine builds it
    the U is the captured one bit for bit; with its lo columns zeroed the layer-1 check must fail"""
    name, cloud, plan, cap = case
    c0 = cloud.size(-1) - 3
    first = engine.sa_fact[0][s][0]
    table = mlp.sa_factor_table(plan.l_xyz[0], cloud.data_ptr() + 12, cloud.size(-1), c0, first.k_pad)
    u = mlp.mlp_dense(table, first, relu=False, a_tf32=True)
    assert torch.equal(_bits(u), _bits(cap.u[0][s])), name
    table[:, c0 + 3:c0 + 6] = 0
    u = mlp.mlp_dense(table, first, relu=False, a_tf32=True)
    bad = types.SimpleNamespace(**vars(cap))
    bad.u = [list(x) for x in cap.u]
    bad.u[0][s] = u
    launch, _, build = R.launches()[2 * s]
    assert launch == f"SA1 scale {s} layer 1"
    with pytest.raises(AssertionError, match="outside the bound") as e:
        R.check_launch(build, bad, plan, cloud, weights, CHUNK, f"[{name}] {launch}, engine without lo")
    print(f"[{name}] {launch} without lo rejected: {str(e.value).split(': ', 1)[1][:80]}")


@pytest.fixture
def cudnn_tf32():
    """the module graph with cuDNN's TF32 on, the reference's (and torch's) default"""
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    yield
    torch.backends.cudnn.allow_tf32 = prev


def test_end_to_end_against_the_f64_twin(case, model, cudnn_tf32):
    """per frame, (mean, 99.9th percentile) of |out - ref64| / mean |ref64|: the engine's within 2x the TF32-operand
    twin's + 1e-6.  The cuDNN-TF32 module graph's is printed for context."""
    name, cloud, plan, cap = case
    b = cloud.size(0)
    m32 = copy.deepcopy(model).eval()
    m64 = copy.deepcopy(model).double().eval()
    m64t = R.tf32_operands(copy.deepcopy(model).double().eval())
    errs = {"engine": [], "tf32 twin": [], "cuDNN TF32": []}
    t0 = time.perf_counter()
    for f0 in range(0, b, CHUNK):
        fr = slice(f0, min(b, f0 + CHUNK))
        log = {k: [] for k in R.DISCRETE}
        g32 = R.module_forward(m32, cloud[fr], R.recorder(log))
        # the twin describes the engine's computation: the module graph chose the engine's centres, balls and 3-NN
        for li in range(4):
            x = plan.l_xyz[li][fr]
            centres = x.gather(1, log["furthest_point_sample"][li].long()[..., None].expand(-1, -1, 3))
            assert torch.equal(_bits(centres), _bits(plan.l_xyz[li + 1][fr])), (name, li)
            for s in range(2):
                assert torch.equal(log["ball_query"][2 * li + s], plan.ball[li][s][fr]), (name, li, s)
            assert torch.equal(log["three_nn"][li][1], plan.nn[3 - li][0][fr]), (name, 3 - li)
        ref64 = R.module_forward(m64, cloud[fr].double(), R.twin(log, True))
        ref_t = R.module_forward(m64t, cloud[fr].double(), R.twin(log, True))
        errs["engine"].append(R.frame_errors(cap.out[fr], ref64))
        errs["tf32 twin"].append(R.frame_errors(ref_t, ref64))
        errs["cuDNN TF32"].append(R.frame_errors(g32, ref64))
        del g32, ref64, ref_t
    e = {k: np.concatenate(v) for k, v in errs.items()}
    for k, v in e.items():
        print(f"[{name}] {k}: per-frame mean {v[:, 0].min():.3g}..{v[:, 0].max():.3g}, "
              f"p99.9 {v[:, 1].min():.3g}..{v[:, 1].max():.3g}")
    ratio = e["engine"] / e["tf32 twin"]
    print(f"[{name}] engine / tf32 twin per frame: mean {ratio[:, 0].min():.3f}..{ratio[:, 0].max():.3f}, "
          f"p99.9 {ratio[:, 1].min():.3f}..{ratio[:, 1].max():.3f}; {time.perf_counter() - t0:.1f} s")
    bad = np.argwhere(e["engine"] > 2 * e["tf32 twin"] + 1e-6)
    assert len(bad) == 0, (name, [(int(f), ("mean", "p99.9")[j], e["engine"][f, j], e["tf32 twin"][f, j])
                                  for f, j in bad[:8]])


def test_batch_invariance(case, engine):
    """every row's arithmetic has a fixed K order and FPS, the ball grid and the 3-NN grid are per frame, so a frame's
    output is the same bits alone, anywhere in the batch and in a batch of reversed order"""
    name, cloud, plan, cap = case
    b = cloud.size(0)
    for f in sorted({0, b // 2, b - 1}):
        one = engine(cloud[f:f + 1].contiguous())
        assert torch.equal(_bits(one[0]), _bits(cap.out[f])), (name, f)
    rev = engine(cloud.flip(0).contiguous())
    assert torch.equal(_bits(rev.flip(0)), _bits(cap.out)), name
