"""The sampled CNN tail without a device: the float64 reference of pvn3d_psp_tail_rows against the module graph it
replaces (this pins the bilinear indices, the zero padding and the BN fold), the layout recognition of
PspTail.from_cnn, and what ptxas makes of the kernel."""
import re

import pytest
import torch

from cnn_tail_cases import SIZES, border_choose, half_map
from pvn3d_b200 import _lib, testing
from pvn3d_b200.cnn_tail import PspTail, fold_tail, sampled_tail_reference
from pvn3d_b200.mlp import _layer_struct, _supported
from test_mlp_sa_fact2_sass_host import _ptxas_props, _sass_functions, compiled  # noqa: F401
from test_mlp_sa_fact2_sass_host import pytestmark as needs_nvcc

KERNEL = "psp_tail_kernel"


@pytest.mark.parametrize("prelu_params", [1, 64])
@pytest.mark.parametrize("h,w", SIZES)
def test_reference_equals_module_graph(h, w, prelu_params):
    cnn = testing.StandInPSPNet(seed=3, prelu_params=prelu_params).double()
    b, n = 2, 300
    x = half_map(b, h, w, seed=h, dtype=torch.float64)
    choose = border_choose(b, n, 2 * h, 2 * w, seed=w)
    with torch.no_grad():
        dense = cnn.final(cnn.up_3(x))                                   # [B, 128, H, W]
    want = torch.gather(dense.flatten(2), 2, choose.repeat(1, 128, 1)).transpose(1, 2).reshape(b * n, 128)
    got, _, _ = sampled_tail_reference(x, choose, fold_tail(cnn, torch.float64))
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())


def test_reference_is_sensitive_to_the_padding():
    # a corner pixel has five taps outside the image: clamping them instead of zeroing must show
    cnn = testing.StandInPSPNet(seed=3).double()
    x = half_map(1, 4, 5, dtype=torch.float64)
    choose = torch.tensor([[[0]]])
    got, _, taps = sampled_tail_reference(x, choose, fold_tail(cnn, torch.float64))
    assert int((taps.view(9, 64).abs().sum(1) == 0).sum()) == 5


def _variants():
    def edit(fn):
        cnn = testing.StandInPSPNet(seed=1)
        fn(cnn)
        return cnn

    up = lambda **kw: torch.nn.Upsample(**{"scale_factor": 2, "mode": "bilinear", "align_corners": True, **kw})  # noqa: E731
    return {
        "align_corners=False": edit(lambda c: c.up_3.conv.__setitem__(0, up(align_corners=False))),
        "nearest": edit(lambda c: c.up_3.conv.__setitem__(0, torch.nn.Upsample(scale_factor=2, mode="nearest"))),
        "scale 4": edit(lambda c: c.up_3.conv.__setitem__(0, up(scale_factor=4))),
        "5x5 conv": edit(lambda c: c.up_3.conv.__setitem__(1, torch.nn.Conv2d(64, 64, 5, padding=2))),
        "stride 2": edit(lambda c: c.up_3.conv.__setitem__(1, torch.nn.Conv2d(64, 64, 3, padding=1, stride=2))),
        "65 channels": edit(lambda c: c.up_3.conv.__setitem__(1, torch.nn.Conv2d(65, 64, 3, padding=1))),
        "ReLU": edit(lambda c: c.up_3.conv.__setitem__(3, torch.nn.ReLU())),
        "no final": edit(lambda c: delattr(c, "final")),
        "final with an activation": edit(lambda c: c.final.append(torch.nn.ReLU())),
        "final 3x3": edit(lambda c: c.final.__setitem__(0, torch.nn.Conv2d(64, 128, 3, padding=1))),
    }


@pytest.mark.parametrize("name", list(_variants()))
def test_other_layouts_are_not_recognised(name):
    assert PspTail.from_cnn(_variants()[name]) is None


def test_stand_in_cnn_of_the_benches_is_not_recognised():
    assert PspTail.from_cnn(testing.StandInCNN()) is None
    assert PspTail.from_cnn(testing.StandInPVN3D(64).cnn) is None


def test_reference_layout_is_recognised_bare_wrapped_and_with_sync_bn():
    cnn = testing.StandInPSPNet(seed=1)
    bare = PspTail.from_cnn(cnn)
    wrapper = torch.nn.Module()
    wrapper.model = cnn
    wrapped = PspTail.from_cnn(wrapper)
    sync = PspTail.from_cnn(torch.nn.SyncBatchNorm.convert_sync_batchnorm(testing.StandInPSPNet(seed=1)))
    for t in (bare, wrapped, sync):
        assert t is not None and t.layer1.w.shape == (64, 576) and t.layer2.w.shape == (128, 64) and t.slope.shape == (64,)
        assert torch.equal(t.layer1.w, bare.layer1.w) and torch.equal(t.layer1.bias, bare.layer1.bias)
    assert wrapped.model is cnn
    assert _supported("pvn3d_psp_tail_supported", bare.layer1, bare.layer2)
    assert not _supported("pvn3d_psp_tail_supported", bare.layer2, bare.layer1)


def test_trunk_is_the_forward_up_to_up_3():
    cnn = testing.StandInPSPNet(seed=2)
    rgb = torch.rand(1, 3, 16, 24)
    with torch.no_grad():
        x_half = PspTail.from_cnn(cnn).trunk(rgb)
        assert x_half.shape == (1, 64, 8, 12)
        assert torch.equal(cnn.final(cnn.up_3(x_half)), cnn(rgb)[0])


def test_entry_points_reject_bad_arguments_before_any_cuda_call():
    import ctypes

    tail = PspTail.from_cnn(testing.StandInPSPNet(seed=1))
    l1, l2 = _layer_struct(tail.layer1), _layer_struct(tail.layer2)
    a1, a2 = ctypes.addressof(l1), ctypes.addressof(l2)
    lib = _lib.load()
    ok = dict(x=4096, b=1, h=4, w=5, choose=4096, n=8, l1=a1, l2=a2, slope=4096, flags=0, out=4096, ldo=256, col0=0)

    def rc(fn="pvn3d_psp_tail_rows", **kw):
        return getattr(lib, fn)(*{**ok, **kw}.values(), None)

    for bad in (dict(x=0), dict(choose=0), dict(slope=0), dict(out=0), dict(h=1), dict(w=1), dict(col0=2), dict(ldo=130),
                dict(col0=132), dict(x=4100), dict(flags=1), dict(b=-1)):
        assert rc(**bad) == -1, bad
    assert rc(fn="pvn3d_psp_tail_rows_bf16", col0=4) == -1
    assert rc(l1=a2, l2=a1) == -2                       # layers of other shapes
    assert rc(h=40000) == -2 and rc(b=2 ** 20, h=2 ** 6, w=2 ** 6) == -2
    assert rc(b=0) == 0 and rc(n=0) == 0                # nothing to do


@needs_nvcc
def test_kernel_has_no_spills_or_serialised_wgmma(compiled):  # noqa: F811
    log, _ = compiled
    props = {k: v for k, v in _ptxas_props(log).items() if KERNEL in k}
    assert len(props) == 2, list(props)                 # f32 rows and bf16 rows
    for name, (regs, st, ld) in props.items():
        assert st == 0 and ld == 0, f"{name}: {regs} registers, {st} B spill stores, {ld} B spill loads"
        assert regs * 544 <= 65536, f"{name}: {regs} registers for 544 threads"
    bad = [line for line in log.splitlines() if re.search(r"C75(19|20)", line) and KERNEL in line]
    assert not bad, "\n".join(bad)


@needs_nvcc
def test_kernel_runs_tf32_hgmma_of_both_widths(compiled):  # noqa: F811
    _, sass = compiled
    funcs = {k: v for k, v in _sass_functions(sass).items() if KERNEL in k}
    assert len(funcs) == 2
    for name, text in funcs.items():
        hgmma = re.findall(r"\bHGMMA\.\S+", text)
        assert hgmma and all(".TF32" in h for h in hgmma), f"{name}: {sorted(set(hgmma))}"
        # layer 1: four m64n64k8 per K chunk (the loop body, and a peeled first chunk); layer 2: eight m64n128k8
        assert len([h for h in hgmma if "64x64x8" in h]) in (4, 8) and len([h for h in hgmma if "64x128x8" in h]) == 8, hgmma
        depbar = len(re.findall(r"\bWARPGROUP\.DEPBAR", text))
        assert 2 * depbar < len(hgmma), f"{name}: {depbar} WARPGROUP.DEPBAR for {len(hgmma)} HGMMA"
