"""Host-side routing of the mixed-precision (torch.autocast) forms of the PointNet++ grouping / interpolation ops and the
PSPNet backward, without a GPU: `_lib.call` is replaced by a recorder, so these tests check which entry point each
dtype and deterministic-mode combination reaches and with which arguments, and which inputs are refused before any
call.  The kernels themselves are checked in test_amp_ext_gpu.py."""
import types

import pytest
import torch

from pvn3d_b200 import _ext, _lib, deterministic

F16, BF16 = _lib.PVN3D_F16, _lib.PVN3D_BF16
CODES = {torch.float16: F16, torch.bfloat16: BF16}


@pytest.fixture
def calls(monkeypatch):
    """records (entry point, arguments) of every _ext / deterministic call; CPU tensors stand in for device ones"""
    rec = []
    monkeypatch.setattr(_ext, "call", lambda fn, dev, *args: rec.append((fn, args)))
    monkeypatch.setattr(_ext, "_need_cuda", lambda x: None)
    monkeypatch.setattr(_ext, "_ordered", lambda fn, dev, b, n, slots, *args: rec.append((fn, (b, n, slots) + args)))
    monkeypatch.setattr(deterministic, "call", lambda fn, dev, *args: rec.append((fn, args)))
    return rec


@pytest.fixture(params=[False, True], ids=["atomic", "deterministic"])
def det(request):
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(request.param)
    yield request.param
    torch.use_deterministic_algorithms(prev, warn_only=warn)


B, C, N, M, S = 2, 5, 40, 7, 4


def _idx(*shape):
    return torch.zeros(shape, dtype=torch.int32)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_group_points_routes_by_dtype(calls, dtype):
    pts, idx = torch.zeros((B, C, N), dtype=dtype), _idx(B, M, S)
    out = _ext.group_points(pts, idx)
    assert out.dtype == dtype and out.shape == (B, C, M, S)
    (fn, args), = calls
    if dtype == torch.float32:
        assert fn == "pvn3d_group_points" and args == (pts.data_ptr(), idx.data_ptr(), B, C, N, M, S, out.data_ptr())
    else:
        assert fn == "pvn3d_group_points_16"
        assert args == (CODES[dtype], pts.data_ptr(), idx.data_ptr(), B, C, N, M, S, out.data_ptr())


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_three_interpolate_routes_by_dtype(calls, dtype):
    pts, idx, w = torch.zeros((B, C, M), dtype=dtype), _idx(B, N, 3), torch.zeros((B, N, 3))
    out = _ext.three_interpolate(pts, idx, w)
    assert out.dtype == dtype and out.shape == (B, C, N)
    (fn, args), = calls
    tail = (pts.data_ptr(), idx.data_ptr(), w.data_ptr(), B, C, M, N, out.data_ptr())
    if dtype == torch.float32:
        assert fn == "pvn3d_three_interpolate" and args == tail
    else:
        assert fn == "pvn3d_three_interpolate_16" and args == (CODES[dtype],) + tail


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_group_points_grad_routes_by_dtype_and_mode(calls, det, dtype):
    g, idx = torch.zeros((B, C, M, S), dtype=dtype), _idx(B, M, S)
    out = _ext.group_points_grad(g, idx, N)
    assert out.dtype == dtype and out.shape == (B, C, N)
    (fn, args), = calls
    core = (g.data_ptr(), idx.data_ptr(), B, C, N, M, S)
    if dtype == torch.float32:
        want = "pvn3d_group_points_grad_ordered" if det else "pvn3d_group_points_grad"
        assert fn == want
        assert args == ((B, N, M * S) if det else ()) + core + (out.data_ptr(),)
    elif det:
        assert fn == "pvn3d_group_points_grad_ordered_16"
        assert args == (B, N, M * S, CODES[dtype]) + core + (out.data_ptr(),)
    else:
        assert fn == "pvn3d_group_points_grad_16"
        assert args[:len(core) + 1] == (CODES[dtype],) + core and args[-1] == out.data_ptr()
        assert args[-2] not in (0, out.data_ptr(), g.data_ptr())          # the float32 scratch


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_three_interpolate_grad_routes_by_dtype_and_mode(calls, det, dtype):
    g, idx, w = torch.zeros((B, C, N), dtype=dtype), _idx(B, N, 3), torch.zeros((B, N, 3))
    out = _ext.three_interpolate_grad(g, idx, w, M)
    assert out.dtype == dtype and out.shape == (B, C, M)
    (fn, args), = calls
    core = (g.data_ptr(), idx.data_ptr(), w.data_ptr(), B, C, N, M)
    if dtype == torch.float32:
        assert fn == ("pvn3d_three_interpolate_grad_ordered" if det else "pvn3d_three_interpolate_grad")
        assert args == ((B, M, 3 * N) if det else ()) + core + (out.data_ptr(),)
    elif det:
        assert fn == "pvn3d_three_interpolate_grad_ordered_16"
        assert args == (B, M, 3 * N, CODES[dtype]) + core + (out.data_ptr(),)
    else:
        assert fn == "pvn3d_three_interpolate_grad_16"
        assert args[:len(core) + 1] == (CODES[dtype],) + core and args[-1] == out.data_ptr()
        assert args[-2] not in (0, out.data_ptr(), g.data_ptr())


BAD = [torch.float64, torch.int32, torch.int64, torch.uint8]


@pytest.mark.parametrize("dtype", BAD)
def test_other_feature_dtypes_are_refused_with_the_usual_text(calls, dtype):
    with pytest.raises(RuntimeError, match="^points must be a float tensor$"):
        _ext.group_points(torch.zeros((B, C, N), dtype=dtype), _idx(B, M, S))
    with pytest.raises(RuntimeError, match="^grad_out must be a float tensor$"):
        _ext.group_points_grad(torch.zeros((B, C, M, S), dtype=dtype), _idx(B, M, S), N)
    with pytest.raises(RuntimeError, match="^points must be a float tensor$"):
        _ext.three_interpolate(torch.zeros((B, C, M), dtype=dtype), _idx(B, N, 3), torch.zeros((B, N, 3)))
    with pytest.raises(RuntimeError, match="^grad_out must be a float tensor$"):
        _ext.three_interpolate_grad(torch.zeros((B, C, N), dtype=dtype), _idx(B, N, 3), torch.zeros((B, N, 3)), M)
    assert calls == []


@pytest.mark.parametrize("wdtype", [torch.float16, torch.bfloat16, torch.float64])
@pytest.mark.parametrize("fdtype", [torch.float32, torch.float16, torch.bfloat16])
def test_weight_stays_float32(calls, fdtype, wdtype):
    with pytest.raises(RuntimeError, match="^weight must be a float tensor$"):
        _ext.three_interpolate(torch.zeros((B, C, M), dtype=fdtype), _idx(B, N, 3), torch.zeros((B, N, 3), dtype=wdtype))
    with pytest.raises(RuntimeError, match="^weight must be a float tensor$"):
        _ext.three_interpolate_grad(torch.zeros((B, C, N), dtype=fdtype), _idx(B, N, 3),
                                    torch.zeros((B, N, 3), dtype=wdtype), M)
    assert calls == []


@pytest.mark.parametrize("idtype", [torch.int64, torch.int16, torch.float16])
def test_idx_stays_int32(calls, idtype):
    with pytest.raises(RuntimeError, match="^idx must be an int tensor$"):
        _ext.group_points(torch.zeros((B, C, N), dtype=torch.bfloat16), torch.zeros((B, M, S), dtype=idtype))
    with pytest.raises(RuntimeError, match="^idx must be an int tensor$"):
        _ext.three_interpolate_grad(torch.zeros((B, C, N), dtype=torch.float16), torch.zeros((B, N, 3), dtype=idtype),
                                    torch.zeros((B, N, 3)), M)
    assert calls == []


def test_out_of_scope_ops_stay_float32(calls):
    """gather_points(_grad) and the coordinate ops keep the float32-only contract"""
    with pytest.raises(RuntimeError, match="^points must be a float tensor$"):
        _ext.gather_points(torch.zeros((B, C, N), dtype=torch.bfloat16), _idx(B, M))
    with pytest.raises(RuntimeError, match="^grad_out must be a float tensor$"):
        _ext.gather_points_grad(torch.zeros((B, C, M), dtype=torch.float16), _idx(B, M), N)
    with pytest.raises(RuntimeError, match="^points must be a float tensor$"):
        _ext.furthest_point_sampling(torch.zeros((B, N, 3), dtype=torch.float16), 4)
    assert calls == []


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16, torch.float64])
def test_deterministic_ordered_accepts_16_bit(monkeypatch, dtype):
    g = types.SimpleNamespace(is_cuda=True, dtype=dtype, dim=lambda: 4)
    torch.use_deterministic_algorithms(True)
    try:
        assert deterministic._ordered(g) == (dtype != torch.float64)
    finally:
        torch.use_deterministic_algorithms(False)
    assert not deterministic._ordered(g)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_psp_backward_routes_by_dtype(calls, monkeypatch, dtype):
    monkeypatch.setattr(deterministic, "_ordered", lambda g: True)
    x = torch.zeros((2, 3, 12, 10), dtype=dtype)
    g = torch.zeros((2, 3, 6, 5), dtype=dtype)
    gi, _ = deterministic._AdaptiveAvgPool2d.backward(types.SimpleNamespace(saved_tensors=(x,)), g)
    ctx = types.SimpleNamespace(scales=(2.0, 2.0), in_size=tuple(x.shape), align=True)
    gu = deterministic._UpsampleBilinear2d.backward(ctx, torch.zeros((2, 3, 24, 20), dtype=dtype))[0]
    assert gi.dtype == dtype and gu.dtype == dtype and gi.shape == gu.shape == x.shape
    (fp, pa), (fu, ua) = calls
    lead = () if dtype == torch.float32 else (CODES[dtype],)
    sfx = "" if dtype == torch.float32 else "_16"
    assert fp == "pvn3d_adaptive_avg_pool2d_backward" + sfx and pa[:len(lead)] == lead
    assert pa[len(lead) + 1:] == (6, 12, 10, 6, 5, gi.data_ptr())
    assert fu == "pvn3d_upsample_bilinear2d_backward" + sfx and ua[:len(lead)] == lead
    assert ua[len(lead) + 1:] == (6, 12, 10, 24, 20, 1, 2.0, 2.0, gu.data_ptr())


def test_16_bit_entry_points_are_bound():
    names = ["pvn3d_group_points_16", "pvn3d_group_points_grad_16", "pvn3d_group_points_grad_ordered_16",
             "pvn3d_three_interpolate_16", "pvn3d_three_interpolate_grad_16",
             "pvn3d_three_interpolate_grad_ordered_16", "pvn3d_adaptive_avg_pool2d_backward_16",
             "pvn3d_upsample_bilinear2d_backward_16"]
    for nm in names:
        assert nm in _lib.EXPORTED_SYMBOLS
        assert _lib._SIGNATURES[nm][1][0] is _lib.c_int          # the dtype code comes first
    assert (F16, BF16) == (1, 2)


def test_unknown_dtype_code_is_refused_before_any_launch():
    """every _16 entry point returns PVN3D_ERR_INVALID_ARG for a code other than PVN3D_F16 / PVN3D_BF16, before it
    looks at its pointers (null here) or touches the device"""
    lib = _lib.load()
    for code in (0, 3, -1, 32):
        assert lib.pvn3d_group_points_16(code, None, None, 1, 1, 1, 1, 1, None, None) == -1
        assert lib.pvn3d_group_points_grad_16(code, None, None, 1, 1, 1, 1, 1, None, None, None) == -1
        assert lib.pvn3d_group_points_grad_ordered_16(code, None, None, 1, 1, 1, 1, 1, None, None, 0, None) == -1
        assert lib.pvn3d_three_interpolate_16(code, None, None, None, 1, 1, 1, 1, None, None) == -1
        assert lib.pvn3d_three_interpolate_grad_16(code, None, None, None, 1, 1, 1, 1, None, None, None) == -1
        assert lib.pvn3d_three_interpolate_grad_ordered_16(code, None, None, None, 1, 1, 1, 1, None, None, 0,
                                                           None) == -1
        assert lib.pvn3d_adaptive_avg_pool2d_backward_16(code, None, 1, 2, 2, 1, 1, None, None) == -1
        assert lib.pvn3d_upsample_bilinear2d_backward_16(code, None, 1, 2, 2, 4, 4, 0, 0.0, 0.0, None, None) == -1
    # a known code with an empty shape returns before any CUDA call too
    assert lib.pvn3d_group_points_16(F16, None, None, 0, 1, 1, 1, 1, None, None) == -1      # null pointers
    assert lib.pvn3d_adaptive_avg_pool2d_backward_16(BF16, None, 0, 2, 2, 1, 1, None, None) == 0
