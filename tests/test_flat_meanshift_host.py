"""Flat mean shift and the clustered ICP refiner, host side (no GPU): the oracle against the sklearn
goldens, the C-ABI binding table and header, argument checks, and make_icp_batch's stray blobs."""
import hashlib
import os

import numpy as np
import pytest

from oracle import flat_meanshift_oracle as fmo
from pvn3d_b200 import _lib, icp, meanshift, synth

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "flat_ms_cases.npz")
HEADER = os.path.join(os.path.dirname(HERE), "include", "pvn3d_b200.h")
NAMES = ("pvn3d_flat_ms_fit_batch", "pvn3d_icp_clustered_workspace_bytes", "pvn3d_icp_refine_batch_clustered")


def golden_cases():
    z = np.load(GOLDEN)
    for k, name in enumerate(z["names"]):
        p = f"c{k}_"
        yield (str(name), z[p + "X"], float(z[p + "bw"]), z[p + "centers"], z[p + "labels"], int(z[p + "n_iter"]))


def test_goldens_cover_the_documented_cases():
    cases = {c[0]: c for c in golden_cases()}
    assert len(cases) == 8 and os.path.getsize(GOLDEN) < 1 << 20
    assert len(cases["cap_4096"][1]) == _lib.FLAT_MS_MAX_PTS and len(cases["ten_points"][1]) == 10
    X, bw = cases["sparse_seeds_are_points"][1:3]
    assert len(fmo.bin_seeds(X, bw)) == len(X)                       # the seeds = X fallback
    assert len(cases["large_split"][3]) > 2                           # an object split into clusters
    counts = np.bincount(cases["equal_count_blobs"][4])
    assert counts.tolist() == [300, 300]                              # the order is decided by the centre
    assert cases["bandwidth_0.03"][2] == 0.03


@pytest.mark.parametrize("case", list(golden_cases()), ids=lambda c: c[0])
def test_oracle_reproduces_sklearn(case):
    name, X, bw, C, L, it = case
    Co, Lo, ito = fmo.flat_mean_shift(X, bw)
    assert ito == it and np.array_equal(Lo, L)
    assert Co.shape == C.shape and np.abs(Co - C).max() <= 1e-12


def test_bin_keys_round_half_to_even():
    bw = 0.0625
    X = np.array([[0.5, 1.5, -0.5], [2.5, -1.5, 0.0], [0.4, 1.6, -0.4]]) * bw
    keys = np.round(X / bw)
    assert keys[:2].tolist() == [[0.0, 2.0, -0.0], [2.0, -2.0, 0.0]]
    S = fmo.bin_seeds(X, bw)
    assert S.dtype == np.float32 and len(S) == 2                      # rows 0 and 2 share a bin


def test_flat_ms_symbols_in_binding_table_and_header():
    header = open(HEADER).read()
    for name in NAMES:
        assert name in _lib._SIGNATURES and f"{name}(" in header
    assert "#define PVN3D_FLAT_MS_MAX_PTS 4096" in header and _lib.FLAT_MS_MAX_PTS == 4096


def _lib_or_skip():
    try:
        return _lib.load()
    except _lib.Pvn3dError:
        pytest.skip("kernel library not built")


def test_flat_ms_argument_checks_launch_nothing():
    lib = _lib_or_skip()
    bad = 0x1000          # never dereferenced: every call below must return before any launch
    before = lib.pvn3d_launch_count()
    args = lambda n_fits, cap, bw, it: (bad, bad, n_fits, cap, bw, it, bad, bad, bad, bad, bad, 0)
    assert lib.pvn3d_flat_ms_fit_batch(*args(3, 4097, 0.06, 300)) == -2          # over the cap
    assert lib.pvn3d_flat_ms_fit_batch(*args(3, 100, 0.0, 300)) == -1            # bandwidth <= 0
    assert lib.pvn3d_flat_ms_fit_batch(*args(3, 100, -0.06, 300)) == -1
    assert lib.pvn3d_flat_ms_fit_batch(*args(3, 100, float("nan"), 300)) == -1
    assert lib.pvn3d_flat_ms_fit_batch(*args(3, 100, 0.06, -1)) == -1            # max_iter < 0
    assert lib.pvn3d_flat_ms_fit_batch(*args(-1, 100, 0.06, 300)) == -1
    assert lib.pvn3d_flat_ms_fit_batch(*args(0, 100, 0.06, 300)) == 0            # nothing to do
    assert lib.pvn3d_icp_clustered_workspace_bytes(16, 12288, 22, 4097) == 0
    assert lib.pvn3d_icp_clustered_workspace_bytes(16, 12288, 22, 2000) > lib.pvn3d_icp_workspace_bytes(16, 12288, 22, 2000)
    ws = (bad & ~255) + 256
    common = (bad, bad, bad, 2, 100, 5)
    rc = lib.pvn3d_icp_refine_batch_clustered(*common, bad, bad, 4097, 10, 20, 1e-9, 0.06, 300, bad, bad, bad, bad, bad,
                                              ws, 1 << 40, 0)
    assert rc == -2
    rc = lib.pvn3d_icp_refine_batch_clustered(*common, bad, bad, 2000, 10, 20, 1e-9, 0.0, 300, bad, bad, bad, bad, bad,
                                              ws, 1 << 40, 0)
    assert rc == -1
    rc = lib.pvn3d_icp_refine_batch_clustered(*common, bad, bad, 2000, 10, 20, 1e-9, 0.06, 300, bad, bad, bad, bad, 0,
                                              ws, 1 << 40, 0)
    assert rc == -1                                                               # cluster_pts_out required
    assert lib.pvn3d_launch_count() == before


def test_python_argument_checks():
    models = {1: np.zeros((4, 3))}
    with pytest.raises(ValueError, match="max_pts"):
        icp.IcpRefiner(models, 2, 1, 100, device="cuda:0", max_pts=4097, min_pts=10, cluster_bandwidth=0.06)
    with pytest.raises(ValueError, match="cluster_bandwidth"):
        icp.IcpRefiner(models, 2, 1, 100, device="cuda:0", max_pts=50, min_pts=10, cluster_bandwidth=0.0)
    with pytest.raises(ValueError, match="cluster_bandwidth"):
        icp.IcpRefiner(models, 2, 1, 100, device="cuda:0", max_pts=50, min_pts=10, cluster_bandwidth=-1.0)
    with pytest.raises(ValueError, match="at most"):
        meanshift.flat_mean_shift(np.zeros((4097, 3)), 0.06)
    with pytest.raises(ValueError):
        meanshift.flat_mean_shift(np.zeros((10, 2)), 0.06)
    with pytest.raises(RuntimeError, match="CUDA only"):
        icp.get_cld_bigest_clus(np.zeros((10, 3)), device="cpu")


def _digest(d):
    h = hashlib.sha256()
    for k in ("pcld", "mask", "gt", "init", "present", "extents"):
        h.update(np.ascontiguousarray(d[k]).tobytes())
    for m in d["models"][1:]:
        h.update(m.tobytes())
    return h.hexdigest()


def test_make_icp_batch_without_strays_is_unchanged():
    # digest of this call's output before n_stray existed
    d = synth.make_icp_batch(4, 5, 700, seed=3, outlier_frac=0.1, n_bg=300, n_stray=0)
    assert _digest(d) == "b2484b3180b0cab54251efa600c83205990fd2a1d90eda8df77872593982a141"


def test_make_icp_batch_stray_blobs():
    d = synth.make_icp_batch(2, 3, 500, seed=3, n_bg=100, n_stray=120)
    assert d["pcld"].shape == (2, 3 * 620 + 100, 3)
    for b in range(2):
        for c in np.nonzero(d["present"][b])[0]:
            pts = d["pcld"][b][d["mask"][b] == c].astype(np.float64)
            assert len(pts) == 620
            X = pts @ d["gt"][b, c, :, :3] - d["gt"][b, c, :, 3] @ d["gt"][b, c, :, :3]   # object frame
            far = np.abs(X) > 0.5 * d["extents"][c] + 0.01
            assert far.any(1).sum() >= 120                            # the blob lies off the box
