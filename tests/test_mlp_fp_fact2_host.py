"""Which factored FP modules pvn3d_mlp_fp_fact2 (the skip term and the second layer of FP1 in one launch) takes, decided
on the host by the library itself (no device needed), the errors of the entry point that leave nothing launched, and
the engine's FP1 choice."""
import ctypes

import pytest
import torch

from pvn3d_b200 import _lib, mlp, testing


def _layers(ks, ns, n2):
    g = torch.Generator().manual_seed(ks + ns + n2)
    ls = mlp.PackedLayer(torch.randn(ns, ks, generator=g), torch.randn(ns, generator=g))
    l2 = mlp.PackedLayer(torch.randn(n2, ns, generator=g), torch.randn(n2, generator=g), ls.n_pad)
    return ls, l2


@pytest.mark.parametrize("widths,fits", [
    ((12, 128, 128), True),     # FP1: 6 features + hi / lo coordinates -> 128 -> 128
    ((32, 128, 128), True),     # a full 32-column table
    ((6, 120, 120), True),      # narrower layers pad to 128
    ((40, 128, 128), False),    # a table wider than one K chunk
    ((12, 256, 128), False),    # a 256-column first layer
    ((12, 128, 256), False),    # a 256-column second layer
    ((12, 64, 64), False),      # 64-column layers
])
def test_fp_fact2_coverage(widths, fits):
    assert mlp.fp_fact2_fits(*_layers(*widths)) is fits


def _call(lib, ls, l2, w_offset=0, p_offset=0, flags=0):
    ok = 0x1000           # never dereferenced: every call below must return before any launch
    s1 = _lib.MlpLayer(ok + w_offset, ok, ls.k_pad, ls.n_pad)
    s2 = _lib.MlpLayer(ok, ok, l2.k_pad, l2.n_pad)
    # p, table, nn_idx, nn_w, b, n_unknown, m_known, layer_s, layer2, flags, out, stream
    return lib.pvn3d_mlp_fp_fact2(ok + p_offset, ok, ok, ok, 2, 1000, 64, ctypes.addressof(s1), ctypes.addressof(s2), flags,
                                  ok, None)


def test_fp_fact2_refuses_without_launching():
    lib = _lib.load()
    before = lib.pvn3d_launch_count()
    assert _call(lib, *_layers(12, 256, 128)) == -2                # PVN3D_ERR_UNSUPPORTED
    assert _call(lib, *_layers(40, 128, 128)) == -2
    assert _call(lib, *_layers(12, 128, 128), w_offset=4) == -1    # PVN3D_ERR_INVALID_ARG: w not 16-byte aligned
    assert _call(lib, *_layers(12, 256, 128), w_offset=4) == -1    # ... checked before the shape
    assert _call(lib, *_layers(12, 128, 128), p_offset=8) == -1    # P not 16-byte aligned
    assert _call(lib, *_layers(12, 128, 128), flags=1) == -1       # a flag other than PVN3D_MLP_RESERVE_SMS
    assert lib.pvn3d_launch_count() == before


def test_supported_query_takes_null_layers():
    ls, l2 = _layers(12, 128, 128)
    s = _lib.MlpLayer(0x1000, 0x1000, ls.k_pad, ls.n_pad)
    assert _lib.load().pvn3d_mlp_fp_fact2_supported(ctypes.addressof(s), None) == 0


def test_engine_runs_fp1_as_p_then_one_fused_launch():
    eng = mlp.FusedPointnet2MSG(testing.seeded_pointnet2msg(0, 1), device="cpu")
    lk, ls, l2 = eng.fp1
    assert (lk.k, lk.n, ls.k, ls.k_pad, ls.n, l2.n) == (256, 128, 12, 32, 128, 128)
    assert mlp.fp_fact2_fits(ls, l2)
    # the skip columns are read through the SA1 factor table: same width as the table
    assert ls.k_pad == eng.sa_fact[0][0][0].k_pad


def test_engine_refuses_an_fp1_the_fused_kernel_does_not_take(monkeypatch):
    monkeypatch.setattr(mlp, "fp_fact2_fits", lambda *args: False)
    with pytest.raises(ValueError, match="FP1"):
        mlp.FusedPointnet2MSG(testing.seeded_pointnet2msg(0, 1), device="cpu")
