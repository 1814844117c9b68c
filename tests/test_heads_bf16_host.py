"""The bf16 heads without a device: weight packing, the argument checks of the bf16 entry points (they refuse before any
launch), the header / binding table, and which precision the PVN3D.forward patch picks under autocast."""
import ctypes

import pytest
import torch

from pvn3d_b200 import _lib, compat, heads, mlp

from test_abi import declared_symbols

OK = 0x1000   # never dereferenced: every call below must return before any launch
BF16_SYMBOLS = ("pvn3d_mlp_dense_bf16", "pvn3d_mlp_dense_frame_bias_bf16", "pvn3d_mlp_dense_sum32_bf16",
                "pvn3d_mlp_fp_fact2_rows_bf16", "pvn3d_gather_pixel_rows_bf16")
RELU, OUT_BF16 = 1, 8


def _rne_bf16_bits(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> bf16 bit patterns, round to nearest even, by integer arithmetic (finite inputs)"""
    i = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    return ((i + 0x7FFF + ((i >> 16) & 1)) >> 16) & 0xFFFF


def test_bf16_packing_rounds_to_nearest_even_and_pads_with_zeros():
    g = torch.Generator().manual_seed(0)
    w = torch.randn(22, 130, generator=g)
    # exact ties: halfway between two bf16 values, one with an even and one with an odd last mantissa bit
    w[0, :4] = torch.tensor([1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -(1.0 + 2 ** -8), 1.0 + 2 ** -8 + 2 ** -20])
    bias = torch.randn(22, generator=g)
    pl = mlp.PackedLayer(w, bias, precision="bf16")
    assert pl.w.dtype == torch.bfloat16 and pl.w.is_contiguous()
    assert (pl.n_pad, pl.k_pad) == (32, 192) and pl.k_pad % 64 == 0
    got = pl.w.view(torch.int16).to(torch.int64) & 0xFFFF
    assert torch.equal(got[:22, :130], _rne_bf16_bits(w))
    assert float(pl.w[0, 0]) == 1.0 and float(pl.w[0, 1]) == 1.0 + 2 ** -6 and float(pl.w[0, 2]) == -1.0
    assert float(pl.w[0, 3]) == 1.0 + 2 ** -7
    assert not bool(pl.w[22:].float().any()) and not bool(pl.w[:, 130:].float().any())
    assert pl.bias.dtype == torch.float32 and torch.equal(pl.bias[:22], bias) and not bool(pl.bias[22:].any())
    # the K of a layer fed by a wider activation: the producer's padded width, rounded up to 64
    assert mlp.PackedLayer(torch.randn(16, 100), torch.zeros(16), 128, precision="bf16").k_pad == 128
    assert mlp.PackedLayer(torch.randn(16, 100), torch.zeros(16), precision="tf32").k_pad == 128
    with pytest.raises(ValueError, match="precision"):
        mlp.PackedLayer(w, bias, precision="fp16")


def test_head_layers_pack_to_bf16_k_multiples_of_64():
    dense_fusion, seg, kpof, ctrof = heads.reference_layout_modules(22, 8)
    pls = [mlp.PackedLayer(*mlp.fold_conv_bn(blk), precision="bf16") for s in (seg, kpof, ctrof) for blk in s.children()]
    assert all(p.k_pad % 64 == 0 and p.w.dtype == torch.bfloat16 for p in pls)


def test_header_declares_the_bf16_entry_points_and_the_binding_has_them():
    declared = declared_symbols()
    for name in BF16_SYMBOLS:
        assert name in declared and name in _lib.EXPORTED_SYMBOLS, name


def _dense(fn, lib, a=OK, lda=1280, a_cols=256, rows=4096, w=OK, bias=OK, k_pad=256, n_pad=1024, flags=RELU | OUT_BF16,
           out=OK, ldo=1280, col0=256, rpf=None):
    if fn == "pvn3d_mlp_dense_frame_bias_bf16":
        return getattr(lib, fn)(a, lda, a_cols, rows, 4096 if rpf is None else rpf, w, bias, k_pad, n_pad, flags, out, ldo,
                                col0, None)
    return getattr(lib, fn)(a, lda, a_cols, rows, w, bias, k_pad, n_pad, flags, out, ldo, col0, None)


@pytest.mark.parametrize("fn", ["pvn3d_mlp_dense_bf16", "pvn3d_mlp_dense_frame_bias_bf16", "pvn3d_mlp_dense_sum32_bf16"])
def test_dense_bf16_refuses_without_launching(fn):
    lib = _lib.load()
    store = fn != "pvn3d_mlp_dense_sum32_bf16"
    flags = RELU | OUT_BF16 if store else RELU
    before = lib.pvn3d_launch_count()
    for kw in ({"a": 0}, {"w": 0}, {"bias": 0}, {"out": 0},
               {"a": OK + 8}, {"w": OK + 8}, {"out": OK + 8},          # not 16-byte aligned
               {"lda": 1284}, {"a_cols": 252}, {"lda": 128},           # lda, a_cols not multiples of 8; lda < a_cols
               {"k_pad": 288}, {"k_pad": 0}, {"n_pad": 1032}, {"n_pad": 0},   # k_pad % 64, n_pad % 16
               {"ldo": 1282}, {"col0": 2}, {"col0": -4}, {"col0": 260},       # col0 + n_pad > ldo
               {"rows": -1}, {"flags": flags | 2}, {"flags": flags | 4}):      # TF32-only flags
        assert _dense(fn, lib, **{"flags": flags, **kw}) == -1, kw
    if not store:
        assert _dense(fn, lib, flags=RELU | OUT_BF16) == -1                    # the sums are fp32
    if fn == "pvn3d_mlp_dense_frame_bias_bf16":
        assert _dense(fn, lib, rpf=1000) == -1                                 # rows_per_frame % 128
        assert _dense(fn, lib, rpf=0) == -1
        assert _dense(fn, lib, rows=4096 + 128, rpf=4096) == -1                # rows % rows_per_frame
    assert _dense(fn, lib, flags=flags, rows=0) == 0                           # nothing to do: no launch either
    assert lib.pvn3d_launch_count() == before


def _gather(lib, emb=OK, emb_bf16=0, b=2, c=128, hw=19200, choose=OK, n=4096, out=OK, ldo=1280, col0=0):
    return lib.pvn3d_gather_pixel_rows_bf16(emb, emb_bf16, b, c, hw, choose, n, out, ldo, col0, None)


def test_gather_bf16_refuses_without_launching():
    lib = _lib.load()
    before = lib.pvn3d_launch_count()
    for kw in ({"emb": 0}, {"choose": 0}, {"out": 0}, {"emb_bf16": 2},
               {"out": OK + 8}, {"choose": OK + 4}, {"emb": OK + 2}, {"emb": OK + 1, "emb_bf16": 1},
               {"c": 124}, {"ldo": 1276}, {"col0": 4}, {"col0": -8}, {"col0": 1160},   # multiples of 8; col0 + c > ldo
               {"hw": 0}, {"b": -1}):
        assert _gather(lib, **kw) == -1, kw
    assert _gather(lib, emb=OK + 2, emb_bf16=1, b=0) == 0                # a 2-byte aligned bf16 map passes the checks
    assert _gather(lib, b=1 << 16, n=1 << 15) == -2                      # B * N = 2^31
    assert _gather(lib, c=264, ldo=1280) == -2                           # C beyond the kernel's 256
    assert _gather(lib, b=0) == 0
    assert lib.pvn3d_launch_count() == before


def _fp1_layers():
    g = torch.Generator().manual_seed(0)
    ls = mlp.PackedLayer(torch.randn(128, 12, generator=g), torch.randn(128, generator=g))
    l2 = mlp.PackedLayer(torch.randn(128, 128, generator=g), torch.randn(128, generator=g), ls.n_pad)
    return ls, l2


def _rows(lib, ls, l2, out=OK, ldo=1280, col0=128, flags=0, bias2=OK, p=OK):
    s1 = _lib.MlpLayer(OK, OK, ls.k_pad, ls.n_pad)
    s2 = _lib.MlpLayer(OK, bias2, l2.k_pad, l2.n_pad)
    return lib.pvn3d_mlp_fp_fact2_rows_bf16(p, OK, OK, OK, 2, 1000, 64, ctypes.addressof(s1), ctypes.addressof(s2), flags,
                                            out, ldo, col0, None)


def test_fp_fact2_rows_bf16_refuses_without_launching():
    lib = _lib.load()
    ls, l2 = _fp1_layers()
    wide = mlp.PackedLayer(torch.randn(256, 12), torch.randn(256))
    before = lib.pvn3d_launch_count()
    for kw in ({"col0": 1160}, {"col0": -8}, {"col0": 4}, {"ldo": 1284}, {"out": OK + 8}, {"out": 0},
               {"bias2": OK + 4}, {"p": OK + 8}, {"flags": 1}):
        assert _rows(lib, ls, l2, **kw) == -1, kw
    assert _rows(lib, wide, l2) == -2                    # a module the kernel does not cover
    assert lib.pvn3d_launch_count() == before


def test_fused_engines_refuse_an_unknown_precision():
    with pytest.raises(ValueError, match="precision"):
        mlp.check_precision("fp16")


@pytest.mark.parametrize("enabled,dtype,want", [(False, torch.bfloat16, "tf32"), (True, torch.bfloat16, "bf16"),
                                                (True, torch.float16, "tf32"), (False, torch.float16, "tf32")])
def test_autocast_precision(monkeypatch, enabled, dtype, want):
    """bf16 autocast on CUDA selects the bf16 heads; fp16 autocast and no autocast keep the TF32 engine"""
    monkeypatch.setattr(torch, "is_autocast_enabled", lambda device_type=None: enabled and device_type == "cuda")
    monkeypatch.setattr(torch, "get_autocast_dtype", lambda device_type: dtype)
    assert compat.autocast_precision() == want


def test_engine_cache_is_per_device_and_precision(monkeypatch):
    import pvn3d_b200.network as network

    built = []

    class Engine:
        def __init__(self, model, device, precision):
            built.append((device, precision))

    monkeypatch.setattr(network, "FusedPVN3D", Engine)
    m = torch.nn.Linear(2, 2)
    e_tf32, e_bf16 = compat.fused_engine(m, "dev0"), compat.fused_engine(m, "dev0", "bf16")
    assert e_tf32 is not e_bf16
    assert compat.fused_engine(m, "dev0", "tf32") is e_tf32 and compat.fused_engine(m, "dev0", "bf16") is e_bf16
    assert built == [("dev0", "tf32"), ("dev0", "bf16")]
    assert sorted(m.__dict__["_pvn3d_b200_engines"]) == [("dev0", "bf16"), ("dev0", "tf32")]
