"""Which SA scales pvn3d_mlp_sa_fact2w (the wide-last-layer variant of the fused layer 2 + layer 3 + max-pool kernel)
takes, decided on the host by the library itself (no device needed): the engine routes a scale to it only when this
says yes, and the entry point refuses every other shape with PVN3D_ERR_UNSUPPORTED before it launches anything."""
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
    ((128, 196, 256), 16, True), ((128, 196, 256), 32, True),     # SA3
    ((256, 256, 512), 16, True), ((256, 384, 512), 32, True),     # SA4
    ((128, 196, 256), 8, False),       # nsample 8
    ((64, 96, 128), 32, False),        # last layer of 128 columns: pvn3d_mlp_sa_fact2's
    ((512, 256, 512), 16, False),      # 16 layer-2 K chunks: the A tile alone would take 128 KB
    ((256, 1024, 512), 16, False),     # A + H tiles (64 + 256 KB) beyond shared memory
])
def test_sa_fact2w_coverage(widths, ns, fits):
    _, l2, l3 = _layers(*widths)
    assert mlp.sa_fact2w_fits(l2, l3, ns) is fits


def test_sa_fact2_and_sa_fact2w_cover_disjoint_scales():
    for widths, ns in [((16, 16, 32), 16), ((64, 96, 128), 32), ((128, 196, 256), 16), ((256, 384, 512), 32)]:
        _, l2, l3 = _layers(*widths)
        assert not (mlp.sa_fact2_fits(l2, l3, ns) and mlp.sa_fact2w_fits(l2, l3, ns))


@pytest.mark.parametrize("widths,ns", [((128, 196, 256), 8), ((256, 1024, 512), 16)])
def test_sa_fact2w_refuses_uncovered_shapes_without_launching(widths, ns):
    first, l2, l3 = _layers(*widths)
    b, n, m = 1, 64, 8
    u = torch.zeros((b * n, first.n_pad))
    v = torch.zeros((b * m, first.n_pad))
    idx = torch.zeros((b, m, ns), dtype=torch.int32)
    out = torch.zeros((b * m, l3.n_pad))
    s2, s3 = mlp._layer_struct(l2), mlp._layer_struct(l3)
    rc = _lib.load().pvn3d_mlp_sa_fact2w(u.data_ptr(), v.data_ptr(), first.n_pad, first.n_pad, idx.data_ptr(), b, n, m, ns,
                                         ctypes.addressof(s2), ctypes.addressof(s3), 0, ns, out.data_ptr(), l3.n_pad, 0, None)
    assert rc == -2      # PVN3D_ERR_UNSUPPORTED
