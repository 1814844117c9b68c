"""Model and inputs of the whole-network tests (tests/test_network_gpu.py) and of tests/golden/network_ref.npz."""
import numpy as np
import torch

from pvn3d_b200 import synth, testing

# (B, N) of the comparison against the reference's PVN3D.forward
NETWORK_CASES = [(2, 4096), (1, 12288)]
IMG_H, IMG_W = 120, 160


def network_model(n):
    """StandInPVN3D for N points (CPU, eval): the weights every network test and the golden use"""
    return testing.StandInPVN3D(n, seed=5)


def network_inputs(b, n):
    """pointcloud [b,n,9] (synthetic LineMOD-like frames), rgb [b,3,IMG_H,IMG_W], choose [b,1,n] int64, on the CPU"""
    frames = synth.make_batch("linemod", b, n_points=n, config_id=4, lm_obj_id=1)
    pc = torch.from_numpy(np.stack([f.cld_rgb_nrm for f in frames])).contiguous()
    rgb = torch.rand(b, 3, IMG_H, IMG_W, generator=torch.Generator().manual_seed(n + b))
    return pc, rgb, testing.sample_choose(b, n, IMG_H * IMG_W, seed=n)


def network_points(n):
    """the point columns of the outputs stored in tests/golden/network_ref.npz"""
    return np.sort(np.random.default_rng(n + 1).choice(n, size=min(n, 384), replace=False))
