"""Hot path A end to end (Pointnet2MSG mirror on the sm_90a ops) against features recorded from the
REFERENCE Pointnet2MSG (tests/golden/pn2msg.npz), and the FramePipeline on synthetic frames."""
import os

import numpy as np
import pytest
import torch

from pvn3d_b200 import synth, testing
from pvn3d_b200.pipeline import FramePipeline

pytestmark = pytest.mark.gpu


def test_pointnet2msg_matches_reference_features(cuda_dev, golden_dir):
    z = np.load(os.path.join(golden_dir, "pn2msg.npz"))
    model = testing.seeded_pointnet2msg(0, 1).to(cuda_dev)
    x = torch.from_numpy(z["cld_rgb_nrm"])[None].to(cuda_dev)
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            y = model(x)[0]
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    got = y[:, torch.from_numpy(z["cols"]).long().to(cuda_dev)].cpu().numpy()
    want = z["feats"]
    # fp32 MLPs on both sides, identical indices: only summation order differs (1e-4 of the feature scale)
    scale = float(z["feat_abs_mean"])
    assert np.abs(got - want).max() <= 2e-3 * max(scale, 1.0), np.abs(got - want).max()
    assert np.abs(got - want).mean() <= 1e-4 * max(scale, 1.0)


@pytest.mark.parametrize("engine", ["fused", "modules"])
@pytest.mark.parametrize("shape,batch", [("linemod", 2), ("ycb", 2)])
def test_frame_pipeline_recovers_synthetic_poses(cuda_dev, shape, batch, engine):
    n = 4096
    frames = synth.make_batch(shape, batch, n_points=n, config_id=9)
    pipe = FramePipeline(shape, batch, n_points=n, device=cuda_dev, engine=engine,
                         lm_obj_id=frames[0].obj_id if shape == "linemod" else 1)
    hb = FramePipeline.pin_batch(synth.stack(frames))
    poses, present = pipe.run_host(hb)
    torch.cuda.synchronize()
    assert pipe.features.shape == (batch, 128, n)
    poses = poses.numpy()
    for bi, f in enumerate(frames):
        if shape == "linemod" and f.obj_id != frames[0].obj_id:
            continue
        for ci, c in enumerate(f.cls_ids):
            assert present[bi, int(c)] == 1
            gt = f.RTs[ci]
            # votes carry 5 mm noise: the recovered translation must land within a few mm
            assert np.linalg.norm(poses[bi, int(c)][:, 3] - gt[:, 3]) < 0.01
            assert np.linalg.norm(poses[bi, int(c)][:, :3] - gt[:, :3]) < 0.2


def test_lookahead_pipeline_equals_serial_pipeline(cuda_dev):
    """the geometry plan of batch i+1 computed on a side stream under the MLPs of batch i (run_device(next_cloud=),
    run_host(hb, next_hb)) must not change a single bit of the features or the poses"""
    n, b = 4096, 3
    batches = [synth.stack(synth.make_batch("ycb", b, n_points=n, config_id=20 + j)) for j in range(4)]
    serial = FramePipeline("ycb", b, n_points=n, device=cuda_dev, overlap=False)
    ahead = FramePipeline("ycb", b, n_points=n, device=cuda_dev, overlap=True, fps_chunk=2)
    dev = [{k: torch.from_numpy(np.ascontiguousarray(v)).to(cuda_dev) for k, v in hb.items()} for hb in batches]
    want = []
    for d in dev:
        p, pr = serial.run_device(d["cld_rgb_nrm"], d["pcld"], d["labels"], d["ctr_of"], d["kp_of"])
        want.append((serial.features.clone(), p.clone(), pr.clone()))
    for j, d in enumerate(dev):
        nxt = dev[j + 1]["cld_rgb_nrm"] if j + 1 < len(dev) else None
        p, pr = ahead.run_device(d["cld_rgb_nrm"], d["pcld"], d["labels"], d["ctr_of"], d["kp_of"], next_cloud=nxt)
        torch.cuda.synchronize()
        assert torch.equal(ahead.features, want[j][0]), j
        assert torch.equal(p, want[j][1]) and torch.equal(pr, want[j][2]), j
    # host path: uploads of the next batch + plan under the current one; a wrong prediction falls back cleanly
    pinned = [FramePipeline.pin_batch(hb) for hb in batches]
    order = [0, 1, 2, 3, 1]
    for j, bi in enumerate(order):
        nxt = pinned[order[j + 1]] if j + 1 < len(order) and j != 2 else (pinned[0] if j == 2 else None)   # j == 2 mispredicts
        p, pr = ahead.run_host(pinned[bi], nxt)
        torch.cuda.synchronize()
        assert torch.equal(ahead.features, want[bi][0]), (j, bi)
        assert torch.equal(p.to(cuda_dev), want[bi][1]) and torch.equal(pr.to(cuda_dev), want[bi][2]), (j, bi)
