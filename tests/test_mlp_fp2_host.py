"""Which FP modules pvn3d_mlp_fp2 (both layers of a two-layer FP module in one launch) takes, decided on the host by the
library itself (no device needed), the errors of the entry point that leave nothing launched, and the engine's
per-module choice."""
import copy
import ctypes

import pytest
import torch

from pvn3d_b200 import _lib, mlp, testing


def _layers(k, n1, n2):
    g = torch.Generator().manual_seed(k + n1 + n2)
    l1 = mlp.PackedLayer(torch.randn(n1, k, generator=g), torch.randn(n1, generator=g))
    l2 = mlp.PackedLayer(torch.randn(n2, n1, generator=g), torch.randn(n2, generator=g), l1.n_pad)
    return l1, l2


@pytest.mark.parametrize("widths,fits", [
    ((1024 + 512, 512, 512), True),    # FP4
    ((512 + 256, 512, 512), True),     # FP3
    ((512 + 96, 256, 256), True),      # FP2
    ((130, 256, 128), True),           # an odd layer-2 block: the second warpgroup sits layer 2 out
    ((256 + 6, 128, 128), False),      # FP1: a 128-column first layer (one block: no pair of warpgroups)
    ((768, 384, 384), False),          # three layer-1 blocks
    ((768, 1024, 512), False),         # the layer-1 tile alone would take 256 KB
    ((768, 512, 200), False),          # a layer-2 width that is not whole 128-column blocks
])
def test_fp2_coverage(widths, fits):
    assert mlp.fp2_fits(*_layers(*widths)) is fits


def _call(lib, l1, l2, w_offset=0):
    ok = 0x1000           # never dereferenced: every call below must return before any launch
    s1 = _lib.MlpLayer(ok + w_offset, ok, l1.k_pad, l1.n_pad)
    s2 = _lib.MlpLayer(ok, ok, l2.k_pad, l2.n_pad)
    c2 = l1.k - 32
    # known_feat, c2, nn_idx, nn_w, skip, lds, c1, b, n_unknown, m_known, layer1, layer2, flags, out, ldo, col0, stream
    return lib.pvn3d_mlp_fp2(ok, c2, ok, ok, ok, 32, 32, 2, 1000, 64, ctypes.addressof(s1), ctypes.addressof(s2), 1, ok,
                             l2.n_pad, 0, None)


def test_fp2_refuses_without_launching():
    lib = _lib.load()
    before = lib.pvn3d_launch_count()
    assert _call(lib, *_layers(768, 384, 384)) == -2          # PVN3D_ERR_UNSUPPORTED
    assert _call(lib, *_layers(768, 1024, 512)) == -2
    assert _call(lib, *_layers(768, 512, 512), w_offset=4) == -1   # PVN3D_ERR_INVALID_ARG: w not 16-byte aligned
    assert _call(lib, *_layers(768, 384, 384), w_offset=4) == -1   # ... checked before the shape
    assert lib.pvn3d_launch_count() == before


def test_engine_runs_fp2_to_fp4_as_one_launch_each():
    eng = mlp.FusedPointnet2MSG(testing.seeded_pointnet2msg(0, 1), device="cpu")
    assert sorted(eng.fp) == [1, 2, 3]
    assert [(l1.k, l1.n, l2.n) for l1, l2 in (eng.fp[i] for i in (1, 2, 3))] == [(608, 256, 256), (768, 512, 512),
                                                                                  (1536, 512, 512)]
    assert all(mlp.fp2_fits(*eng.fp[i]) for i in (1, 2, 3))


def test_engine_refuses_a_module_the_fused_kernel_does_not_take(monkeypatch):
    monkeypatch.setattr(mlp, "fp2_fits", lambda *args: False)
    with pytest.raises(ValueError, match="FP2"):
        mlp.FusedPointnet2MSG(testing.seeded_pointnet2msg(0, 1), device="cpu")


def test_engine_refuses_an_fp_module_with_other_than_two_layers():
    model = testing.seeded_pointnet2msg(0, 1)
    model.FP_modules[2].mlp.add_module("layer2", copy.deepcopy(model.FP_modules[2].mlp.layer1))   # 512 -> 512 again
    with pytest.raises(ValueError, match="FP3"):
        mlp.FusedPointnet2MSG(model, device="cpu")
