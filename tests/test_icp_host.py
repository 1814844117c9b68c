"""ICP refinement, host side (no GPU): the oracle against the reference goldens, the scene-point
selection rule, IcpRefiner argument checks and the C-ABI binding table."""
import os

import numpy as np
import pytest

from oracle import icp_oracle
from pvn3d_b200 import _lib, icp

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "icp_cases.npz")


def golden_cases():
    z = np.load(GOLDEN)
    for k, name in enumerate(z["names"]):
        p = f"c{k}_"
        yield (str(name), z[p + "A"], z[p + "B"], z[p + "init"] if bool(z[p + "has_init"]) else None,
               int(z[p + "max_iter"]), float(z[p + "tol"]), z[p + "T"], z[p + "dist"], int(z[p + "i"]))


def test_goldens_cover_the_documented_cases():
    names = [c[0] for c in golden_cases()]
    assert len(names) == 8
    z = np.load(GOLDEN)
    assert z["c5_i"] == 29 and z["c5_tol"] == 0.0          # the cap is hit
    assert len(z["c6_A"]) >= 10000 and len(z["c7_A"]) == 10
    assert os.path.getsize(GOLDEN) < 1 << 20


@pytest.mark.parametrize("case", list(golden_cases()), ids=lambda c: c[0])
def test_oracle_reproduces_reference(case):
    name, A, B, init, it, tol, T, dist, i = case
    To, do, io = icp_oracle.my_icp(A, B, init, max_iterations=it, tolerance=tol)
    assert io == i
    assert np.abs(To - T).max() < 1e-12
    assert np.abs(do - dist).max() < 1e-12


def test_selection_rule():
    mask = np.array([0, 3, 3, 1, 3, 3, 3, 0, 3, 3], np.int32)   # class 3 at 1,2,4,5,6,8,9 (cnt 7)
    assert icp_oracle.select(mask, 3, 3).tolist() == [1, 4, 6]  # positions floor(j*7/3) = 0, 2, 4
    assert icp_oracle.select(mask, 3, 7).tolist() == [1, 2, 4, 5, 6, 8, 9]
    assert icp_oracle.select(mask, 3, 100).tolist() == [1, 2, 4, 5, 6, 8, 9]
    assert icp_oracle.select(mask, 2, 5).tolist() == []
    big = np.zeros(5000, np.int32)
    big[::2] = 4                                                   # 2500 points of class 4
    sel = icp_oracle.select(big, 4, 2000)
    assert len(sel) == 2000 and np.all(np.diff(sel) > 0) and sel[0] == 0


def test_oracle_nearest_lowest_index_on_ties():
    pts = np.array([[0, 0, 0], [1, 0, 0], [0, 0, 0], [1, 0, 0]], np.float64)
    d, i = icp_oracle.nearest(np.array([[0.5, 0, 0], [2, 0, 0], [-1, 0, 0]]), pts)
    assert i.tolist() == [0, 1, 0] and d.tolist() == [0.5, 1.0, 1.0]


def test_model_table():
    pts, off = icp.model_table({1: np.ones((4, 3)), 3: np.zeros((2, 3))}, 5)
    assert pts.dtype == np.float32 and pts.shape == (6, 3)
    assert off.tolist() == [0, 0, 4, 4, 6, 6]
    pts, off = icp.model_table([np.ones((9, 3)), np.ones((4, 3)), None], 3)   # class 0 is never a model
    assert off.tolist() == [0, 0, 4, 4]
    with pytest.raises(ValueError):
        icp.model_table({5: np.ones((4, 3))}, 5)
    with pytest.raises(ValueError):
        icp.model_table({1: np.ones((4, 2))}, 5)


def test_refiner_argument_checks():
    models = {1: np.zeros((4, 3))}
    with pytest.raises(TypeError):
        icp.IcpRefiner(models, 2, 1, 100, device="cuda")                      # max_pts / min_pts required
    with pytest.raises(RuntimeError, match="CUDA only"):
        icp.IcpRefiner(models, 2, 1, 100, max_pts=50, min_pts=10, device="cpu")
    with pytest.raises(RuntimeError, match="CUDA only"):
        icp.my_icp(np.zeros((4, 3)), np.zeros((4, 3)), device="cpu")


def test_icp_symbols_in_binding_table():
    for name in ("pvn3d_icp_models_bytes", "pvn3d_icp_build_models", "pvn3d_icp_workspace_bytes",
                 "pvn3d_icp_refine_batch", "pvn3d_icp_fit"):
        assert name in _lib._SIGNATURES
