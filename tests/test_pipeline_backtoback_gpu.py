"""FramePipeline's look-ahead schedule run the way bench.py runs it: steps issued back to back, no host
synchronisation between them, at the benchmark's shapes (LineMOD 32 x 12288: the MLPs of SA1-2 leave SMs to the
sampler, reserve_levels 2; YCB 16 x 12288 and stress 8 x 49152: every level does, reserve_levels 5).

With a synchronise after every step no ordering mistake between step i's kernels and step i+1's uploads, sampling or
allocator reuse can show; here each step's outputs are clone()d on the current stream (stream-ordered, so legal) and
everything is compared after ONE final synchronise, bit for bit, with a serial pipeline (overlap=False).

This is one deterministic pass.  A race need not show on a given run: a pass is necessary evidence, not a proof.  If a
step differs, that is the finding -- read the event and stream ordering in pipeline.py against it.
"""
import numpy as np
import pytest
import torch

import bench
from pvn3d_b200 import synth
from pvn3d_b200.pipeline import FramePipeline

pytestmark = pytest.mark.gpu
KEYS = ("cld_rgb_nrm", "pcld", "labels", "ctr_of", "kp_of")


def _host_batches(name, count):
    cfg = bench.CONFIGS[name]
    kw = dict(lm_obj_id=1) if cfg["shape"] == "linemod" else {}
    if cfg.get("n_inst"):
        kw["n_instances"] = cfg["n_inst"]
    return cfg, [synth.stack(synth.make_batch(cfg["shape"], cfg["batch"], n_points=cfg["n_points"], config_id=40 + j, **kw))
                 for j in range(count)]


def _pipe(cfg, dev, **kw):
    return FramePipeline(cfg["shape"], cfg["batch"], n_points=cfg["n_points"], device=dev, lm_obj_id=1, **kw)


def _serial_results(cfg, dev_batches, dev):
    serial = _pipe(cfg, dev, overlap=False)
    want = []
    for d in dev_batches:
        p, pr = serial.run_device(*(d[k] for k in KEYS))
        want.append((serial.features.clone(), p.clone(), pr.clone()))
    torch.cuda.synchronize()
    # the batches must be told apart: a step answering with its neighbour's result has to show
    assert not torch.equal(want[0][0], want[1][0]) and not torch.equal(want[0][1], want[1][1])
    return want


def _same(got, want):
    return (torch.equal(got[0].view(torch.int32), want[0].view(torch.int32)) and torch.equal(got[1].view(torch.int32),
            want[1].view(torch.int32)) and torch.equal(got[2], want[2]))


@pytest.mark.parametrize("name,steps,reserve_levels", [("linemod", 8, 2), ("ycb", 8, 5), ("stress", 3, 5)])
def test_lookahead_steps_back_to_back_equal_serial(cuda_dev, name, steps, reserve_levels):
    nb = min(4, steps)
    cfg, host = _host_batches(name, nb)
    dev = [{k: torch.from_numpy(np.ascontiguousarray(v)).to(cuda_dev) for k, v in hb.items()} for hb in host]
    want = _serial_results(cfg, dev, cuda_dev)
    order = [j % nb for j in range(steps)]                        # 0,1,2,3,0,1,2,3
    for kw in (dict(), dict(fps_chunk=5), dict(pose_stream=False)):
        ahead = _pipe(cfg, cuda_dev, overlap=True, **kw)
        assert ahead.reserve_levels == reserve_levels
        assert ahead.fps_chunk == (5 if kw.get("fps_chunk") else cfg["batch"])     # 5 divides no benchmark batch
        got = []
        for j, bi in enumerate(order):
            d = dev[bi]
            nxt = dev[order[(j + 1) % steps]]["cld_rgb_nrm"]      # always named, as bench.Runner.step_device does:
            p, pr = ahead.run_device(*(d[k] for k in KEYS), next_cloud=nxt)        # a non-zero SM reserve every step
            got.append((ahead.features.clone(), p.clone(), pr.clone()))
        torch.cuda.synchronize()
        for j, bi in enumerate(order):
            assert _same(got[j], want[bi]), (name, kw, "step", j, "batch", bi)
        # a warmed step makes no host synchronisation
        torch.cuda.set_sync_debug_mode("error")
        try:
            d = dev[order[0]]
            ahead.run_device(*(d[k] for k in KEYS), next_cloud=dev[order[1]]["cld_rgb_nrm"])
        finally:
            torch.cuda.set_sync_debug_mode("default")
        torch.cuda.synchronize()
        del ahead, got


def test_run_host_back_to_back_keeps_result_i_until_call_i_plus_2(cuda_dev):
    """run_host(hb, next_hb) eight times without a device-wide synchronise; the pinned result of call i is read only
    after call i+1 has been issued, waiting on an event recorded after call i.  Call 2 names the wrong next batch and
    batch 3 is run twice in a row."""
    cfg, host = _host_batches("ycb", 4)
    dev = [{k: torch.from_numpy(np.ascontiguousarray(v)).to(cuda_dev) for k, v in hb.items()} for hb in host]
    want = _serial_results(cfg, dev, cuda_dev)
    pinned = [FramePipeline.pin_batch(hb) for hb in host]
    ahead = _pipe(cfg, cuda_dev, overlap=True)
    order = [0, 1, 2, 3, 3, 0, 1, 2]
    named = [1, 2, 0, 3, 0, 1, 2, None]                           # named[2] = 0 but call 3 runs batch 3: a misprediction
    events, results, feats, read = [], [], [], {}

    def read_back(i):
        events[i].synchronize()                                   # this call's work only, not the device
        read[i] = (results[i][0].clone(), results[i][1].clone())

    for j, bi in enumerate(order):
        results.append(ahead.run_host(pinned[bi], None if named[j] is None else pinned[named[j]]))
        feats.append(ahead.features.clone())
        ev = torch.cuda.Event()
        ev.record()
        events.append(ev)
        if j >= 1:
            read_back(j - 1)
    read_back(len(order) - 1)
    torch.cuda.synchronize()
    for j, bi in enumerate(order):
        got = (feats[j], read[j][0].to(cuda_dev), read[j][1].to(cuda_dev))
        assert _same(got, want[bi]), ("call", j, "batch", bi)
