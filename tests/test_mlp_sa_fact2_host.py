"""Which SA scales pvn3d_mlp_sa_fact2 takes, decided on the host by the library itself (no device needed): the
engine routes a scale to the fused kernel only when this says yes, and the entry point refuses every other shape
with PVN3D_ERR_UNSUPPORTED before it launches anything."""
import ctypes

import pytest
import torch

from pvn3d_b200 import _lib, mlp


def _layers(n1, n2, n3):
    g = torch.Generator().manual_seed(n1 + n2 + n3)
    first = mlp.PackedLayer(torch.randn(n1, 9, generator=g), torch.zeros(n1))
    l2 = mlp.PackedLayer(torch.randn(n2, n1, generator=g), torch.randn(n2, generator=g), first.n_pad)
    l3 = mlp.PackedLayer(torch.randn(n3, n2, generator=g), torch.randn(n3, generator=g), l2.n_pad)
    return first, l2, l3


@pytest.mark.parametrize("widths,ns,fits", [
    ((16, 16, 32), 16, True), ((32, 32, 64), 32, True), ((64, 64, 128), 16, True), ((64, 96, 128), 32, True),   # SA1, SA2
    ((256, 64, 128), 16, True),        # more layer-2 K chunks (8) than ring stages (5)
    ((128, 196, 256), 16, False),      # SA3: last layer wider than 128
    ((32, 32, 64), 8, False),          # nsample 8
    ((1024, 128, 128), 16, False),     # W2 alone (512 KB) exceeds shared memory
])
def test_sa_fact2_coverage(widths, ns, fits):
    _, l2, l3 = _layers(*widths)
    assert mlp.sa_fact2_fits(l2, l3, ns) is fits


def test_sa_fact2_refuses_uncovered_shapes_without_launching():
    first, l2, l3 = _layers(1024, 128, 128)
    b, n, m, ns = 1, 64, 8, 16
    u = torch.zeros((b * n, first.n_pad))
    v = torch.zeros((b * m, first.n_pad))
    idx = torch.zeros((b, m, ns), dtype=torch.int32)
    out = torch.zeros((b * m, l3.n_pad))
    s2, s3 = mlp._layer_struct(l2), mlp._layer_struct(l3)
    rc = _lib.load().pvn3d_mlp_sa_fact2(u.data_ptr(), v.data_ptr(), first.n_pad, first.n_pad, idx.data_ptr(), b, n, m, ns,
                                        ctypes.addressof(s2), ctypes.addressof(s3), 0, ns, out.data_ptr(), l3.n_pad, 0, None)
    assert rc == -2      # PVN3D_ERR_UNSUPPORTED
