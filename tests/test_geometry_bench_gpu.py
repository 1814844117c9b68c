"""The geometry plan FusedPointnet2MSG computes (sampled centres, both ball tables per SA level, 3-NN indices and
weights per FP level) against oracle/pn2 at the three shapes bench.py runs: LineMOD 32 x 12288, YCB 16 x 12288 and the
stress configuration 8 x 49152, built exactly as bench.Runner builds them.

Every frame of every configuration is checked (the C oracle needs a few seconds per configuration on eight cores).
The oracle is chained on its OWN previous level and the comparison goes level by level, so a wrong index is reported
at the level where it happens.  Each bit-exact comparison is paired with the mutants of tests/geo_ref.py it rejects
on the same data.  The benchmark's level 0 of the stress configuration is the generic sampling kernel (49152 > 12288
points) at m = 2048; its ball query scans 384 boxes; its FP1 3-NN is the x-sorted walk at 49152 x 2048.
"""
import numpy as np
import pytest
import torch

import bench
import geo_ref as G
from helpers import t
from oracle import pn2
from pvn3d_b200 import mlp, synth, testing
from pvn3d_b200.pointnet2 import SA_SPEC

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine(cuda_dev):
    return mlp.FusedPointnet2MSG(testing.seeded_pointnet2msg(0, 1), cuda_dev)


def bench_cloud(name):
    cfg = bench.CONFIGS[name]
    kw = dict(lm_obj_id=1) if cfg["shape"] == "linemod" else {}
    if cfg.get("n_inst"):
        kw["n_instances"] = cfg["n_inst"]
    frames = synth.make_batch(cfg["shape"], cfg["batch"], n_points=cfg["n_points"], config_id=cfg["config_id"],
                              first_frame=0, **kw)
    return synth.stack(frames)["cld_rgb_nrm"]


def oracle_plan(cloud):
    """-> l_xyz [5], fps idx [4], ball [4][2], nn {i: (idx, d2)} with every level computed from the oracle's previous one"""
    l_xyz, fidx, ball, nn = [np.ascontiguousarray(cloud[..., :3])], [], [], {}
    for npoint, radii, nsamples, _ in SA_SPEC:
        fidx.append(pn2.furthest_point_sampling(l_xyz[-1], npoint))
        l_xyz.append(G.gather_rows(l_xyz[-1], fidx[-1]))
        ball.append([pn2.ball_query(l_xyz[-1], l_xyz[-2], float(np.float32(r)), ns) for r, ns in zip(radii, nsamples)])
    for i in range(4):
        d2, idx = pn2.three_nn(l_xyz[i], l_xyz[i + 1])
        nn[i] = (idx, d2)
    return l_xyz, fidx, ball, nn


@pytest.fixture(scope="module", params=list(bench.CONFIGS))
def case(request, cuda_dev, engine):
    cloud = bench_cloud(request.param)
    dev_cloud = t(cloud, cuda_dev)
    plan = engine.geometry(dev_cloud)
    torch.cuda.synchronize()
    return request.param, cloud, dev_cloud, plan, oracle_plan(cloud)


def test_plan_equals_oracle_level_by_level(case):
    name, cloud, _, plan, (l_xyz, fidx, ball, nn) = case
    for li in range(4):
        got = plan.l_xyz[li + 1].cpu().numpy()
        assert np.array_equal(G.bits(got), G.bits(l_xyz[li + 1])), (name, "centres of level", li + 1)
        assert not np.array_equal(l_xyz[li + 1], G.mut_frame0(l_xyz[li + 1])), (name, li)
        for s in range(2):
            g = plan.ball[li][s].cpu().numpy()
            assert np.array_equal(g, ball[li][s]), (name, "ball", li, s, int((g != ball[li][s]).sum()))
            for mutant in (G.mut_frame0(ball[li][s]), G.mut_ball_pad_zero(ball[li][s]),
                           G.mut_ball_scan_order(ball[li][s], l_xyz[li + 1])):
                assert not np.array_equal(mutant, ball[li][s]), (name, li, s)
    for i in range(4):
        idx, d2 = nn[i]
        g = plan.nn[i][0].cpu().numpy()
        assert np.array_equal(g, idx), (name, "3-NN", i, int((g != idx).sum()))
        assert not np.array_equal(G.mut_frame0(idx), idx)
        w = plan.nn[i][1].cpu().numpy()
        assert G.same_bits(w, G.weights_ref(d2)), (name, "weights", i)
        assert (d2[..., 0] == 0).any()                       # every known point is also a query: 1 / (0 + 1e-8)
        assert not G.same_bits(G.mut_weights_no_eps(d2), G.weights_ref(d2))
        assert G.weights_err_over_bound(w, G.weights_f64(d2)) <= 1.0


def test_chunked_sampling_gives_the_same_centres(case, engine):
    """fps_chunk launches offset raw pointers into the cloud and the index table: 1 frame per launch, 5 (which divides
    none of 32, 16, 8: the last launch is short) and the whole batch"""
    name, cloud, dev_cloud, plan, (l_xyz, _, _, _) = case
    b = cloud.shape[0]
    for k in (1, 5, b):
        p = engine.sampling(dev_cloud, fps_chunk=k)
        for li in range(1, 5):
            assert np.array_equal(G.bits(p.l_xyz[li].cpu().numpy()), G.bits(l_xyz[li])), (name, k, li)
    assert not np.array_equal(l_xyz[1], G.mut_frame0(l_xyz[1]))          # a chunk reading frame 0 would show


def test_plan_on_a_side_stream_under_a_busy_default_stream(case, engine, cuda_dev):
    """what the look-ahead does: the plan computed on a high-priority stream while the default stream runs an unrelated
    large shared-MLP launch"""
    name, cloud, dev_cloud, plan, _ = case
    g = torch.Generator().manual_seed(5)
    layer = mlp.PackedLayer(torch.randn(128, 128, generator=g).to(cuda_dev), torch.zeros(128, device=cuda_dev))
    a = torch.randn(1 << 20, 128, generator=g).to(cuda_dev)
    side = torch.cuda.Stream(cuda_dev, priority=-1)
    torch.cuda.synchronize()
    for _ in range(6):
        mlp.mlp_dense(a, layer)
    with torch.cuda.stream(side):
        p = engine.geometry(dev_cloud, fps_chunk=5)
    torch.cuda.synchronize()
    for li in range(1, 5):
        assert torch.equal(p.l_xyz[li], plan.l_xyz[li]), (name, li)
    for li in range(4):
        assert all(torch.equal(x, y) for x, y in zip(p.ball[li], plan.ball[li])), (name, li)
        assert torch.equal(p.nn[li][0], plan.nn[li][0]) and torch.equal(p.nn[li][1].view(torch.int32),
                                                                          plan.nn[li][1].view(torch.int32)), (name, li)
    assert not torch.equal(plan.ball[0][0], plan.ball[0][0][:1].expand_as(plan.ball[0][0]))


def test_features_from_the_oracle_plan_are_the_engines_features(case, engine, cuda_dev):
    """the number the benchmark dumps: the shared MLPs on a plan assembled from ORACLE tensors give the very bits they
    give on the engine's own plan -- and different bits on a plan with the ball padding mutated"""
    name, cloud, dev_cloud, plan, (l_xyz, _, ball, nn) = case

    def uploaded(ball_tables):
        p = mlp.GeoPlan(dev_cloud, [t(x, cuda_dev) for x in l_xyz])
        p.ball = [tuple(t(x, cuda_dev) for x in lv) for lv in ball_tables]
        p.nn = {i: (t(idx, cuda_dev), t(G.weights_ref(d2), cuda_dev)) for i, (idx, d2) in nn.items()}
        return p

    own = engine.features(dev_cloud, plan)
    assert torch.equal(engine.features(dev_cloud, uploaded(ball)).view(torch.int32), own.view(torch.int32)), name
    wrong = [[G.mut_ball_pad_zero(x) for x in lv] for lv in ball]
    assert not torch.equal(engine.features(dev_cloud, uploaded(wrong)), own), name
