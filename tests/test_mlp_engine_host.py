"""FusedPointnet2MSG's choice of kernels and the shared-MLP entry points' weight-pointer check, on the host (the
kernel library is loaded; no device is needed)."""
import pytest

from pvn3d_b200 import _lib, mlp, testing


def test_engine_routes_every_sa_scale_to_a_fused_kernel():
    eng = mlp.FusedPointnet2MSG(testing.seeded_pointnet2msg(0, 1), device="cpu")
    kernels = [[fused for _, _, fused in scales] for scales in eng.sa]
    assert kernels == [[mlp.mlp_sa_fact2] * 2] * 2 + [[mlp.mlp_sa_fact2w] * 2] * 2


def test_engine_refuses_a_scale_no_fused_kernel_takes(monkeypatch):
    monkeypatch.setattr(mlp, "sa_fact2_fits", lambda *args: False)
    monkeypatch.setattr(mlp, "sa_fact2w_fits", lambda *args: False)
    with pytest.raises(ValueError, match="SA1 scale 0"):
        mlp.FusedPointnet2MSG(testing.seeded_pointnet2msg(0, 1), device="cpu")


def test_misaligned_weights_are_refused_without_launching():
    """the weights are read 16 bytes at a time: a w that is not 16-byte aligned is an invalid argument, for every
    layer kernel"""
    lib = _lib.load()
    ok = 0x1000           # never dereferenced: every call below must return before any launch
    w = ok + 4
    before = lib.pvn3d_launch_count()
    # a, lda, a_cols, rows, w, bias, k_pad, n_pad, flags, pool, out, ldo, col0, stream
    assert lib.pvn3d_mlp_dense(ok, 32, 32, 128, w, ok, 32, 16, 1, 0, ok, 16, 0, None) == -1
    assert lib.pvn3d_mlp_dense(ok, 32, 32, 128, w, ok, 32, 16, 1, 16, ok, 16, 0, None) == -1
    assert lib.pvn3d_mlp_dense(ok, 32, 32, 128, w, ok, 32, 128, 1, 16, ok, 128, 0, None) == -1
    assert lib.pvn3d_mlp_dense_frame_bias(ok, 32, 32, 256, 128, w, ok, 32, 16, 1, ok, 16, 0, None) == -1
    assert lib.pvn3d_mlp_dense_sum32(ok, 32, 32, 128, w, ok, 32, 16, 1, ok, 16, 0, None) == -1
    # known_feat, c2, nn_idx, nn_w, skip, lds, c1, b, n_unknown, m_known, w, bias, k_pad, n_pad, flags, out, ldo, col0
    assert lib.pvn3d_mlp_fp_first(ok, 32, ok, ok, None, 0, 0, 1, 128, 16, w, ok, 32, 16, 1, ok, 16, 0, None) == -1
    # p, s, ld, c_valid, nn_idx, nn_w, b, n_unknown, m_known, w, bias, k_pad, n_pad, flags, out, ldo, col0
    assert lib.pvn3d_mlp_fp_fact(ok, ok, 32, 32, ok, ok, 1, 128, 16, w, ok, 32, 16, 1, ok, 16, 0, None) == -1
    # u, v, ldu, c_valid, idx, b, n, m, ns, w, bias, k_pad, n_pad, flags, pool, out, ldo, col0
    assert lib.pvn3d_mlp_sa_fact(ok, ok, 32, 32, ok, 1, 64, 8, 16, w, ok, 32, 16, 1, 0, ok, 16, 0, None) == -1
    assert lib.pvn3d_mlp_sa_fact(ok, ok, 32, 32, ok, 1, 64, 8, 16, w, ok, 32, 16, 1, 16, ok, 16, 0, None) == -1
    assert lib.pvn3d_launch_count() == before
