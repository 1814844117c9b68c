"""The whole-network forward without a device: the new C entry points refuse bad arguments before any launch, and the
PVN3D.forward patch sends training, grad-enabled and CPU calls to the original forward (on a stand-in class)."""
import ctypes

import pytest
import torch

from pvn3d_b200 import _lib, compat, mlp

OK = 0x1000   # never dereferenced: every call below must return before any launch


def _gather(lib, emb=OK, b=2, c=128, hw=19200, choose=OK, n=4096, out=OK, ldo=1280, col0=0):
    return lib.pvn3d_gather_pixel_rows(emb, b, c, hw, choose, n, out, ldo, col0, None)


def test_gather_refuses_without_launching():
    lib = _lib.load()
    before = lib.pvn3d_launch_count()
    assert _gather(lib, emb=0) == -1                     # null pointers
    assert _gather(lib, choose=0) == -1
    assert _gather(lib, out=0) == -1
    assert _gather(lib, out=OK + 4) == -1                # out not 16-byte aligned
    assert _gather(lib, choose=OK + 4) == -1             # int64 index not 8-byte aligned
    assert _gather(lib, emb=OK + 2) == -1                # emb not 4-byte aligned
    assert _gather(lib, col0=1160) == -1                 # col0 + C > ldo
    assert _gather(lib, col0=-4) == -1
    assert _gather(lib, ldo=1282) == -1                  # ldo not a multiple of 4
    assert _gather(lib, c=126) == -1                     # C not a multiple of 4
    assert _gather(lib, hw=0) == -1
    assert _gather(lib, b=-1) == -1
    assert _gather(lib, b=1 << 16, n=1 << 15) == -2      # B * N = 2^31
    assert _gather(lib, c=260, ldo=1280) == -2           # C beyond the kernel's 256
    assert _gather(lib, b=0) == 0                        # nothing to do: no launch either
    assert lib.pvn3d_launch_count() == before


def _layers():
    g = torch.Generator().manual_seed(0)
    ls = mlp.PackedLayer(torch.randn(128, 12, generator=g), torch.randn(128, generator=g))
    l2 = mlp.PackedLayer(torch.randn(128, 128, generator=g), torch.randn(128, generator=g), ls.n_pad)
    return ls, l2


def _rows(lib, ls, l2, out=OK, ldo=1280, col0=128, flags=0, bias2=OK, p=OK):
    s1 = _lib.MlpLayer(OK, OK, ls.k_pad, ls.n_pad)
    s2 = _lib.MlpLayer(OK, bias2, l2.k_pad, l2.n_pad)
    # p, table, nn_idx, nn_w, b, n_unknown, m_known, layer_s, layer2, flags, out, ldo, col0, stream
    return lib.pvn3d_mlp_fp_fact2_rows(p, OK, OK, OK, 2, 1000, 64, ctypes.addressof(s1), ctypes.addressof(s2), flags,
                                       out, ldo, col0, None)


def test_fp_fact2_rows_refuses_without_launching():
    lib = _lib.load()
    ls, l2 = _layers()
    wide = mlp.PackedLayer(torch.randn(256, 12), torch.randn(256))
    before = lib.pvn3d_launch_count()
    assert _rows(lib, ls, l2, col0=1160) == -1           # col0 + 128 > ldo
    assert _rows(lib, ls, l2, col0=-4) == -1
    assert _rows(lib, ls, l2, col0=2) == -1              # col0 not a multiple of 4
    assert _rows(lib, ls, l2, ldo=1282) == -1            # ldo not a multiple of 4
    assert _rows(lib, ls, l2, out=OK + 8) == -1          # out not 16-byte aligned
    assert _rows(lib, ls, l2, out=0) == -1
    assert _rows(lib, ls, l2, bias2=OK + 4) == -1        # layer-2 bias not 8-byte aligned
    assert _rows(lib, ls, l2, p=OK + 8) == -1            # the checks of pvn3d_mlp_fp_fact2 hold as well
    assert _rows(lib, ls, l2, flags=1) == -1
    assert _rows(lib, wide, l2) == -2                    # a module the kernel does not cover
    assert lib.pvn3d_launch_count() == before


class _Recorder(torch.nn.Module):
    """stands in for the reference PVN3D: its forward records the call"""

    def __init__(self):
        super().__init__()
        self.lin = torch.nn.Linear(2, 2)
        self.calls = 0

    def forward(self, pointcloud, rgb, choose):
        self.calls += 1
        return "original"


@pytest.fixture
def patched():
    cls = type("PatchedRecorder", (_Recorder,), {})
    compat.patch_pvn3d_forward(cls)
    return cls


def test_patch_is_idempotent_and_keeps_the_original(patched):
    fwd = patched.forward
    compat.patch_pvn3d_forward(patched)
    assert patched.forward is fwd and fwd._pvn3d_b200_orig is _Recorder.forward


def test_patch_routes_training_grad_and_cpu_calls_to_the_original(patched, monkeypatch):
    monkeypatch.setattr(compat, "fused_engine", lambda *a: pytest.fail("the fused path must not be taken"))
    m = patched()
    x = torch.zeros(1, 8, 9), torch.zeros(1, 3, 4, 4), torch.zeros(1, 1, 8, dtype=torch.int64)
    m.train()
    with torch.no_grad():
        assert m(*x) == "original"                        # training
    m.eval()
    with torch.enable_grad():
        assert m(*x) == "original"                        # autograd on
    with torch.no_grad():
        assert m(*x) == "original"                        # CPU inputs
    assert m.calls == 3


def test_fused_network_is_cuda_only():
    from pvn3d_b200 import network, testing

    with pytest.raises(RuntimeError, match="CUDA"):
        network.FusedPVN3D(testing.StandInPVN3D(256), device="cpu")
