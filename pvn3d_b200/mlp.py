"""Hot path A on the library's own kernels end to end: FusedPointnet2MSG.

Takes a Pointnet2MSG module (this package's mirror or the reference's -- same state_dict layout),
folds every Conv2d(1x1, no bias) + BatchNorm2d (eval) pair into a TF32-rounded, zero-padded weight
matrix + bias, and runs `Pointnet2MSG.forward` (reference pvn3d/lib/pvn3d.py:126-154) as:

  per SA level : furthest_point_sampling -> ball_query of both radii -> factored first SharedMLP layer:
                 U = W1 . [f | x] once per point (pvn3d_sa_factor_table, shared by both scales, then
                 pvn3d_mlp_dense) and V = W1x . c - b1 once per centre (pvn3d_sa_centre_term) -> layers 2
                 and 3 on relu(U[idx] - V) with ReLU + max-pool over nsample in ONE launch
                 (pvn3d_mlp_sa_fact2 for SA1 / SA2, pvn3d_mlp_sa_fact2w for SA3 / SA4), written straight
                 into the level's point-major feature table
  per FP level : three_nn -> inverse-distance weights ->
                 FP2-4: both layers in ONE launch (pvn3d_mlp_fp2): three_interpolate + concat fused into the
                        tensor-core operand producer, the layer-1 activations kept in shared memory
                 FP1  : factored first layer, P = W1k . known once per known point (pvn3d_mlp_dense) ->
                        S = W1s . skip + b1 and the second layer on relu(interpolated P + S) in ONE launch
                        (pvn3d_mlp_fp_fact2), stored channel-major [B,128,N], the layout the reference returns

The grouped tensors [B,3+C,M,S] and the interpolated tensors [B,C,n] are never materialised; no
cuDNN / cuBLAS / ATen kernel runs in this path.
"""
from __future__ import annotations

import ctypes
from typing import Callable, Dict, List, Tuple

import torch

from . import _ext, _lib
from ._lib import check, ptr
from .pointnet2 import SA_SPEC


def tf32_round(x: torch.Tensor) -> torch.Tensor:
    """round-to-nearest (ties away) to TF32's 10-bit mantissa, like cvt.rna.tf32.f32"""
    i = x.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def fold_conv_bn(layer: torch.nn.Module) -> Tuple[torch.Tensor, torch.Tensor]:
    """layer = Sequential(conv [, normlayer.bn], activation) of SharedMLP (pytorch_utils.py:80-134).
    Returns (W [N,K], bias [N]) with the eval-mode BatchNorm folded in."""
    w = layer.conv.weight.detach().double().flatten(1)
    n = w.size(0)
    bias = layer.conv.bias.detach().double() if layer.conv.bias is not None else torch.zeros(n, dtype=torch.float64, device=w.device)
    if hasattr(layer, "normlayer"):
        bn = layer.normlayer.bn
        scale = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
        w = w * scale[:, None]
        bias = (bias - bn.running_mean.detach().double()) * scale + bn.bias.detach().double()
    return w.float(), bias.float()


class PackedLayer:
    """one folded layer in the layout pvn3d_mlp_* expects"""

    def __init__(self, w: torch.Tensor, bias: torch.Tensor, k_valid_prev_pad: int | None = None):
        n, k = w.shape
        self.n, self.k = n, k
        self.n_pad = (n + 15) // 16 * 16
        k_in = k if k_valid_prev_pad is None else k_valid_prev_pad     # width of the producing activation
        self.k_pad = (max(k, k_in) + 31) // 32 * 32
        wp = torch.zeros((self.n_pad, self.k_pad), dtype=torch.float32, device=w.device)
        wp[:n, :k] = w
        self.w = tf32_round(wp).contiguous()
        self.bias = torch.zeros((self.n_pad,), dtype=torch.float32, device=w.device)
        self.bias[:n] = bias


MLP_RELU, MLP_ROUND_OUT, MLP_A_TF32, MLP_OUT_CN = 1, 2, 4, 16      # include/pvn3d_b200.h PVN3D_MLP_*


def _flags(relu, round_out=False, a_tf32=False, reserve=0):
    """PVN3D_MLP_* flags; reserve = SMs left to concurrent kernels (PVN3D_MLP_RESERVE_SMS)"""
    return ((MLP_RELU if relu else 0) | (MLP_ROUND_OUT if round_out else 0) | (MLP_A_TF32 if a_tf32 else 0)
            | ((int(reserve) & 0xFF) << 8))


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


def mlp_dense(a2d: torch.Tensor, layer: PackedLayer, relu=True, pool=0, out=None, col0=0, round_out=False,
              a_tf32=False, reserve=0):
    """a2d [rows, lda] point-major activations (all lda columns valid or zero).  a_tf32: a2d came out of
    a layer run with round_out=True (values already TF32) -> asynchronous copy path."""
    lib = _lib.load()
    rows, lda = a2d.shape
    if out is None:
        out = torch.empty((rows // pool if pool else rows, layer.n_pad), dtype=torch.float32, device=a2d.device)
    with torch.cuda.device(a2d.device):
        rc = lib.pvn3d_mlp_dense(ptr(a2d), lda, lda, rows, ptr(layer.w), ptr(layer.bias), layer.k_pad, layer.n_pad,
                                 _flags(relu, round_out, a_tf32, reserve), pool, ptr(out), out.size(-1), col0, _stream(a2d.device))
    check(rc, "pvn3d_mlp_dense")
    return out


def mlp_fp_first(known_feat_pm, nn_idx, nn_w, skip_ptr, lds, c1, layer: PackedLayer, relu=True, round_out=False, reserve=0):
    lib = _lib.load()
    b, m_known, c2 = known_feat_pm.shape
    n_unknown = nn_idx.shape[1]
    out = torch.empty((b * n_unknown, layer.n_pad), dtype=torch.float32, device=known_feat_pm.device)
    with torch.cuda.device(known_feat_pm.device):
        rc = lib.pvn3d_mlp_fp_first(ptr(known_feat_pm), c2, ptr(nn_idx), ptr(nn_w), skip_ptr, lds, c1, b, n_unknown,
                                    m_known, ptr(layer.w), ptr(layer.bias), layer.k_pad, layer.n_pad,
                                    _flags(relu, round_out, reserve=reserve), ptr(out), out.size(-1), 0,
                                    _stream(known_feat_pm.device))
    check(rc, "pvn3d_mlp_fp_first")
    return out


def fp2_fits(layer1: PackedLayer, layer2: PackedLayer) -> bool:
    """whether pvn3d_mlp_fp2 takes a two-layer FP module (the library's own rule: a first layer of 256 or 512 columns, a
    second layer of a multiple of 128 columns over exactly those, tiles and stages within shared memory -- FP2-FP4)"""
    l1, l2 = _layer_struct(layer1), _layer_struct(layer2)
    return bool(_lib.load().pvn3d_mlp_fp2_supported(ctypes.addressof(l1), ctypes.addressof(l2)))


def mlp_fp2(known_feat_pm, nn_idx, nn_w, skip_ptr, lds, c1, layer1: PackedLayer, layer2: PackedLayer, out=None, col0=0,
            round_out=False, reserve=0):
    """both layers of an FP module in one launch (pvn3d_mlp_fp2): the same bits as
    mlp_fp_first(.., layer1, round_out=True) -> mlp_dense(.., layer2, a_tf32=True, round_out=round_out)"""
    lib = _lib.load()
    b, m_known, c2 = known_feat_pm.shape
    n_unknown = nn_idx.shape[1]
    if out is None:
        out = torch.empty((b * n_unknown, layer2.n_pad), dtype=torch.float32, device=known_feat_pm.device)
    l1, l2 = _layer_struct(layer1), _layer_struct(layer2)
    with torch.cuda.device(known_feat_pm.device):
        rc = lib.pvn3d_mlp_fp2(ptr(known_feat_pm), c2, ptr(nn_idx), ptr(nn_w), skip_ptr, lds, c1, b, n_unknown, m_known,
                               ctypes.addressof(l1), ctypes.addressof(l2), _flags(True, round_out, reserve=reserve), ptr(out),
                               out.size(-1), col0, _stream(known_feat_pm.device))
    check(rc, "pvn3d_mlp_fp2")
    return out


def sa_factor_table(xyz: torch.Tensor, feat_ptr: int, ldf: int, c_feat: int, k_pad: int) -> torch.Tensor:
    """[B,n,3] coordinates + point-major descriptors -> [B*n, k_pad] rows [tf32(f) | hi(x) | lo(x) | 0] (see
    pvn3d_sa_factor_table in include/pvn3d_b200.h)"""
    lib = _lib.load()
    rows = xyz.size(0) * xyz.size(1)
    out = torch.empty((rows, k_pad), dtype=torch.float32, device=xyz.device)
    with torch.cuda.device(xyz.device):
        rc = lib.pvn3d_sa_factor_table(ptr(xyz), feat_ptr, ldf, c_feat, rows, k_pad, ptr(out), _stream(xyz.device))
    check(rc, "pvn3d_sa_factor_table")
    return out


def sa_centre_term(new_xyz: torch.Tensor, wx: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """V[i] = Wx . c_i - bias for every sampled centre: new_xyz [B,m,3], wx [n_pad,3], bias [n_pad] -> [B*m, n_pad]"""
    lib = _lib.load()
    rows = new_xyz.size(0) * new_xyz.size(1)
    n_pad = wx.size(0)
    out = torch.empty((rows, n_pad), dtype=torch.float32, device=new_xyz.device)
    with torch.cuda.device(new_xyz.device):
        rc = lib.pvn3d_sa_centre_term(ptr(new_xyz), ptr(wx), ptr(bias), rows, n_pad, ptr(out), _stream(new_xyz.device))
    check(rc, "pvn3d_sa_centre_term")
    return out


def mlp_sa_fact(u: torch.Tensor, v: torch.Tensor, idx: torch.Tensor, n: int, layer: PackedLayer, relu=True, pool=0,
                out=None, col0=0, round_out=False, reserve=0):
    """second layer of a factored SA scale: rows relu(U[idx] - V) -> layer (pvn3d_mlp_sa_fact)"""
    lib = _lib.load()
    b, m, ns = idx.shape
    rows = b * m * ns
    if out is None:
        out = torch.empty((rows // pool if pool else rows, layer.n_pad), dtype=torch.float32, device=u.device)
    with torch.cuda.device(u.device):
        rc = lib.pvn3d_mlp_sa_fact(ptr(u), ptr(v), u.size(-1), u.size(-1), ptr(idx), b, n, m, ns, ptr(layer.w), ptr(layer.bias),
                                   layer.k_pad, layer.n_pad, _flags(relu, round_out, reserve=reserve), pool, ptr(out),
                                   out.size(-1), col0, _stream(u.device))
    check(rc, "pvn3d_mlp_sa_fact")
    return out


def _layer_struct(layer: PackedLayer) -> _lib.MlpLayer:
    return _lib.MlpLayer(layer.w.data_ptr(), layer.bias.data_ptr(), layer.k_pad, layer.n_pad)


def sa_fact2_fits(layer2: PackedLayer, layer3: PackedLayer, ns: int) -> bool:
    """whether pvn3d_mlp_sa_fact2 takes the scale (the library's own rule: nsample 16 or 32, both layers at most 128
    columns, weights + layer-2 tile within shared memory -- SA1 and SA2)"""
    l2, l3 = _layer_struct(layer2), _layer_struct(layer3)
    return bool(_lib.load().pvn3d_mlp_sa_fact2_supported(ctypes.addressof(l2), ctypes.addressof(l3), ns))


def mlp_sa_fact2(u: torch.Tensor, v: torch.Tensor, idx: torch.Tensor, n: int, layer2: PackedLayer, layer3: PackedLayer,
                 out=None, col0=0, round_out=False, reserve=0):
    """layers 2 and 3 of a factored SA scale + max-pool over nsample in one launch (pvn3d_mlp_sa_fact2): the same bits
    as mlp_sa_fact(.., layer2, round_out=True) -> mlp_dense(.., layer3, pool=ns, a_tf32=True)"""
    lib = _lib.load()
    b, m, ns = idx.shape
    if out is None:
        out = torch.empty((b * m, layer3.n_pad), dtype=torch.float32, device=u.device)
    l2, l3 = _layer_struct(layer2), _layer_struct(layer3)
    with torch.cuda.device(u.device):
        rc = lib.pvn3d_mlp_sa_fact2(ptr(u), ptr(v), u.size(-1), u.size(-1), ptr(idx), b, n, m, ns, ctypes.addressof(l2),
                                    ctypes.addressof(l3), _flags(True, round_out, reserve=reserve), ns, ptr(out), out.size(-1),
                                    col0, _stream(u.device))
    check(rc, "pvn3d_mlp_sa_fact2")
    return out


def sa_fact2w_fits(layer2: PackedLayer, layer3: PackedLayer, ns: int) -> bool:
    """whether pvn3d_mlp_sa_fact2w takes the scale (the library's own rule: nsample 16 or 32, a last layer wider than
    128 columns, layer-2 K at most 256, A + H tiles + three weight stages within shared memory -- SA3 and SA4)"""
    l2, l3 = _layer_struct(layer2), _layer_struct(layer3)
    return bool(_lib.load().pvn3d_mlp_sa_fact2w_supported(ctypes.addressof(l2), ctypes.addressof(l3), ns))


def mlp_sa_fact2w(u: torch.Tensor, v: torch.Tensor, idx: torch.Tensor, n: int, layer2: PackedLayer, layer3: PackedLayer,
                  out=None, col0=0, round_out=False, reserve=0):
    """mlp_sa_fact2 for a wide last layer (pvn3d_mlp_sa_fact2w: weights streamed, both layers in 128-column blocks):
    the same bits as mlp_sa_fact(.., layer2, round_out=True) -> mlp_dense(.., layer3, pool=ns, a_tf32=True)"""
    lib = _lib.load()
    b, m, ns = idx.shape
    if out is None:
        out = torch.empty((b * m, layer3.n_pad), dtype=torch.float32, device=u.device)
    l2, l3 = _layer_struct(layer2), _layer_struct(layer3)
    with torch.cuda.device(u.device):
        rc = lib.pvn3d_mlp_sa_fact2w(ptr(u), ptr(v), u.size(-1), u.size(-1), ptr(idx), b, n, m, ns, ctypes.addressof(l2),
                                     ctypes.addressof(l3), _flags(True, round_out, reserve=reserve), ns, ptr(out), out.size(-1),
                                     col0, _stream(u.device))
    check(rc, "pvn3d_mlp_sa_fact2w")
    return out


def mlp_fp_fact(p: torch.Tensor, s_: torch.Tensor, nn_idx: torch.Tensor, nn_w: torch.Tensor, m_known: int,
                layer: PackedLayer, relu=True, round_out=False, reserve=0, out_cn=False):
    """second layer of a factored FP module: rows relu(sum_t w_t P[idx_t] + S) -> layer (pvn3d_mlp_fp_fact).
    out_cn: return [b, n_pad, n_unknown] (channel-major frames, PVN3D_MLP_OUT_CN) instead of [b * n_unknown, n_pad]"""
    lib = _lib.load()
    b, n_unknown = nn_idx.shape[0], nn_idx.shape[1]
    ld = p.size(-1)
    shape = (b, layer.n_pad, n_unknown) if out_cn else (b * n_unknown, layer.n_pad)
    out = torch.empty(shape, dtype=torch.float32, device=p.device)
    with torch.cuda.device(p.device):
        rc = lib.pvn3d_mlp_fp_fact(ptr(p), ptr(s_), ld, ld, ptr(nn_idx), ptr(nn_w), b, n_unknown, m_known, ptr(layer.w),
                                   ptr(layer.bias), layer.k_pad, layer.n_pad,
                                   _flags(relu, round_out, reserve=reserve) | (MLP_OUT_CN if out_cn else 0),
                                   ptr(out), layer.n_pad, 0, _stream(p.device))
    check(rc, "pvn3d_mlp_fp_fact")
    return out


def fp_fact2_fits(layer_s: PackedLayer, layer2: PackedLayer) -> bool:
    """whether pvn3d_mlp_fp_fact2 takes a factored FP module (the library's own rule: a skip layer 32 -> 128 over an SA
    factor table, a second layer 128 -> 128 -- FP1)"""
    ls, l2 = _layer_struct(layer_s), _layer_struct(layer2)
    return bool(_lib.load().pvn3d_mlp_fp_fact2_supported(ctypes.addressof(ls), ctypes.addressof(l2)))


def mlp_fp_fact2(p: torch.Tensor, table: torch.Tensor, nn_idx: torch.Tensor, nn_w: torch.Tensor, m_known: int,
                 layer_s: PackedLayer, layer2: PackedLayer, reserve=0):
    """the skip term and the second layer of a factored FP module in one launch (pvn3d_mlp_fp_fact2) -> [b, 128,
    n_unknown]: the same bits as mlp_fp_fact(p, mlp_dense(table, layer_s, relu=False, a_tf32=True), .., layer2,
    out_cn=True)"""
    lib = _lib.load()
    b, n_unknown = nn_idx.shape[0], nn_idx.shape[1]
    assert p.size(-1) == layer_s.n_pad and table.size(-1) == layer_s.k_pad and table.size(0) == b * n_unknown
    out = torch.empty((b, layer2.n_pad, n_unknown), dtype=torch.float32, device=p.device)
    ls, l2 = _layer_struct(layer_s), _layer_struct(layer2)
    with torch.cuda.device(p.device):
        rc = lib.pvn3d_mlp_fp_fact2(ptr(p), ptr(table), ptr(nn_idx), ptr(nn_w), b, n_unknown, m_known,
                                    ctypes.addressof(ls), ctypes.addressof(l2), _flags(False, reserve=reserve), ptr(out),
                                    _stream(p.device))
    check(rc, "pvn3d_mlp_fp_fact2")
    return out


def mlp_fp_fact2_rows(p: torch.Tensor, table: torch.Tensor, nn_idx: torch.Tensor, nn_w: torch.Tensor, m_known: int,
                      layer_s: PackedLayer, layer2: PackedLayer, out: torch.Tensor, col0: int, reserve=0) -> torch.Tensor:
    """mlp_fp_fact2 with its output point-major in columns col0 .. col0+127 of the row table out [b * n_unknown, ldo]
    (pvn3d_mlp_fp_fact2_rows): tf32_round of the transposed [b, 128, n_unknown], bit for bit"""
    lib = _lib.load()
    b, n_unknown = nn_idx.shape[0], nn_idx.shape[1]
    assert p.size(-1) == layer_s.n_pad and table.size(-1) == layer_s.k_pad and table.size(0) == b * n_unknown
    assert out.dim() == 2 and out.size(0) == b * n_unknown and out.stride(1) == 1
    ls, l2 = _layer_struct(layer_s), _layer_struct(layer2)
    with torch.cuda.device(p.device):
        rc = lib.pvn3d_mlp_fp_fact2_rows(ptr(p), ptr(table), ptr(nn_idx), ptr(nn_w), b, n_unknown, m_known,
                                         ctypes.addressof(ls), ctypes.addressof(l2), _flags(False, reserve=reserve), ptr(out),
                                         out.stride(0), col0, _stream(p.device))
    check(rc, "pvn3d_mlp_fp_fact2_rows")
    return out


def three_nn_weights(dist2: torch.Tensor) -> torch.Tensor:
    lib = _lib.load()
    w = torch.empty_like(dist2)
    rows = dist2.numel() // 3
    with torch.cuda.device(dist2.device):
        rc = lib.pvn3d_three_nn_weights(ptr(dist2), rows, ptr(w), _stream(dist2.device))
    check(rc, "pvn3d_three_nn_weights")
    return w


class GeoPlan:
    """the coordinate-only half of one Pointnet2MSG.forward (FusedPointnet2MSG.geometry)"""

    def __init__(self, cloud: torch.Tensor, l_xyz: List[torch.Tensor]):
        self.key = (cloud.data_ptr(), tuple(cloud.shape))
        self.l_xyz = l_xyz                       # xyz of levels 0..4
        self.ball: List[Tuple[torch.Tensor, torch.Tensor]] = []     # per SA level: idx of both radii
        self.nn: Dict[int, Tuple[torch.Tensor, torch.Tensor]] = {}  # per FP level: (idx [B,n,3], weights [B,n,3])
        self.done = None                          # event recorded by whoever computed the plan on a side stream

    def tensors(self):
        for t in self.l_xyz:
            yield t
        # (ball / nn tables are computed on the consumer's stream: FusedPointnet2MSG.queries)


class FusedPointnet2MSG:
    """Inference engine for Pointnet2MSG on libpvn3d_b200 only (see module docstring)."""

    def __init__(self, model: torch.nn.Module, device="cuda"):
        self.dev = torch.device(device)
        model = model.to(self.dev).eval()
        # SA scales: the first layer is evaluated once per POINT instead of once per (centre, neighbour) pair (it is
        # linear before its ReLU; DESIGN.md section 4), layers 2 and 3 + the max-pool run as one launch
        #: per level, per scale: (first layer [W_f | W_x | W_x] with its bias moved into V, Wx [n_pad,3], b1 [n_pad])
        self.sa_fact: List[List[Tuple[PackedLayer, torch.Tensor, torch.Tensor]]] = []
        #: per level, per scale: (layer 2, layer 3, the kernel that runs both and the max-pool)
        self.sa: List[List[Tuple[PackedLayer, PackedLayer, Callable]]] = []
        self.sa_out: List[int] = []
        for li, (sa, (_, _, nsamples, _)) in enumerate(zip(model.SA_modules, SA_SPEC)):
            facts, scales = [], []
            for si, (mlp, ns) in enumerate(zip(sa.mlps, nsamples)):
                w, bias = fold_conv_bn(mlp[0])                    # reference column order [xyz(3) | features]
                wf, wxyz = w[:, 3:], w[:, :3]
                first = PackedLayer(torch.cat([wf, wxyz, wxyz], dim=1), torch.zeros_like(bias))
                n_pad = first.n_pad
                wx = torch.zeros((n_pad, 3), dtype=torch.float32, device=self.dev)
                wx[: w.size(0)] = tf32_round(wxyz.to(self.dev))
                b1 = torch.zeros((n_pad,), dtype=torch.float32, device=self.dev)
                b1[: w.size(0)] = bias.to(self.dev)
                facts.append((first, wx.contiguous(), b1))
                l2 = PackedLayer(*fold_conv_bn(mlp[1]), n_pad)
                l3 = PackedLayer(*fold_conv_bn(mlp[2]), l2.n_pad)
                if sa_fact2_fits(l2, l3, ns):
                    fused = mlp_sa_fact2        # SA1 / SA2: weights resident, layer 2 stays on chip
                elif sa_fact2w_fits(l2, l3, ns):
                    fused = mlp_sa_fact2w       # SA3 / SA4: the same, weights streamed
                else:
                    raise ValueError(f"SA{li + 1} scale {si}: no fused kernel takes layers 2 and 3 "
                                     f"({l2.n} -> {l3.n} channels) at nsample {ns}")
                scales.append((l2, l3, fused))
            self.sa_fact.append(facts)
            self.sa.append(scales)
            self.sa_out.append(sum(l3.n for _, l3, _ in scales))
            assert all(l3.n % 4 == 0 for _, l3, _ in scales)
        #: FP2-FP4 (keys 1-3): (layer 1, layer 2), both run by pvn3d_mlp_fp2 with the interpolation fused into the
        #: operand producer of layer 1
        self.fp: Dict[int, Tuple[PackedLayer, PackedLayer]] = {}
        for i, fp in enumerate(model.FP_modules):
            if i == 0:
                continue
            layers, prev_pad = [], None
            for layer in fp.mlp:
                pl = PackedLayer(*fold_conv_bn(layer), prev_pad)
                prev_pad = pl.n_pad
                layers.append(pl)
            if len(layers) != 2 or not fp2_fits(*layers):
                raise ValueError(f"FP{i + 1}: no fused kernel takes its layers "
                                 f"({' -> '.join(str(x) for x in [layers[0].k] + [l.n for l in layers])} channels)")
            self.fp[i] = (layers[0], layers[1])
        #: FP1, factored: W1 = [W_k (known columns) | W_s (skip columns)] as (P layer W_k, S layer W_s + b1, layer 2).
        #: The skip of FP1 is the raw cloud: W_s reads it through the level-0 factor table [f | hi x | lo x].
        fp1 = model.FP_modules[0].mlp
        w, bias = fold_conv_bn(fp1[0])
        c2 = w.size(1) - (model.SA_modules[0].mlps[0][0].conv.weight.size(1) - 3)
        lk = PackedLayer(w[:, :c2].contiguous(), torch.zeros_like(bias))
        ws = torch.cat([w[:, c2:], torch.zeros((w.size(0), 6), dtype=w.dtype, device=w.device)], dim=1)
        ls = PackedLayer(ws.contiguous(), bias)
        l2 = PackedLayer(*fold_conv_bn(fp1[1]), lk.n_pad) if len(fp1) == 2 else None
        if l2 is None or not fp_fact2_fits(ls, l2):
            raise ValueError(f"FP1: no fused kernel takes its skip term and second layer "
                             f"({len(fp1)} layers, {ws.size(1)} skip columns -> {ls.n} channels)")
        self.fp1 = (lk, ls, l2)
        self._marks = None

    def _m(self, family: str) -> None:
        """profile(): close the interval since the previous mark and charge it to `family`"""
        if self._marks is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self._marks.append((family, e))

    @torch.no_grad()
    def profile(self, pointcloud: torch.Tensor, reps: int = 3) -> Dict[str, float]:
        """One instrumented forward per repetition: CUDA events on the launching stream between the kernel
        families (fps / ball / mlp / three_nn / glue); returns the median ms per family per call.  The
        events serialise nothing that is not already serial (one stream)."""
        import statistics

        self.forward(pointcloud)
        runs = []
        for _ in range(reps):
            torch.cuda.synchronize(self.dev)
            self._marks = []
            self._m("start")
            self.forward(pointcloud)
            marks, self._marks = self._marks, None
            torch.cuda.synchronize(self.dev)
            acc: Dict[str, float] = {}
            for (_, e0), (fam, e1) in zip(marks[:-1], marks[1:]):
                acc[fam] = acc.get(fam, 0.0) + e0.elapsed_time(e1)
            runs.append(acc)
        return {k: statistics.median(r.get(k, 0.0) for r in runs) for k in runs[0]}

    @torch.no_grad()
    def sampling(self, pointcloud: torch.Tensor, fps_chunk: int = 0) -> "GeoPlan":
        """The four furthest-point samplings of Pointnet2MSG.forward and the sampled centres (reference
        pointnet2_modules.py:44-53): 3708 dependent arg-max iterations on ONE CTA per frame -- latency-bound
        and narrow (B of the SMs).  They depend on the coordinates only, so FramePipeline runs them for
        batch i+1 on a side stream under the shared MLPs of batch i.
        fps_chunk > 0: sample that many frames per launch, so that a caller who keeps only `fps_chunk` SMs free
        for this stream never has more sampling CTAs pending than free SMs."""
        assert pointcloud.is_cuda and pointcloud.is_contiguous() and pointcloud.dtype == torch.float32
        b = pointcloud.size(0)
        xyz = pointcloud[..., :3].contiguous()
        self._m("glue")
        plan = GeoPlan(pointcloud, [xyz])
        lib = _lib.load()
        for li, (npoint, radii, nsamples, _) in enumerate(SA_SPEC):
            x = plan.l_xyz[-1]
            if fps_chunk and fps_chunk < b:
                fidx = torch.empty((b, npoint), dtype=torch.int32, device=self.dev)
                n = x.size(1)
                with torch.cuda.device(self.dev):
                    for f0 in range(0, b, fps_chunk):
                        nb = min(fps_chunk, b - f0)
                        check(lib.pvn3d_furthest_point_sampling(x.data_ptr() + f0 * n * 12, nb, n, npoint,
                                                                fidx.data_ptr() + f0 * npoint * 4, _stream(self.dev)),
                              "pvn3d_furthest_point_sampling")
            else:
                fidx = _ext.furthest_point_sampling(x, npoint)
            self._m("fps")
            plan.l_xyz.append(_ext.gather_xyz(x, fidx))
            self._m("glue")
        return plan

    @torch.no_grad()
    def queries(self, plan: "GeoPlan") -> "GeoPlan":
        """The wide coordinate-only kernels: ball queries of both radii of every SA level and the 3-NN indices +
        inverse-distance weights of every FP level (pointnet2_modules.py:57-60,183-186).  They fill the machine,
        so they run on the stream of the MLPs (0.9 ms per 32-frame batch)."""
        for li, (npoint, radii, nsamples, _) in enumerate(SA_SPEC):
            plan.ball.append(_ext.ball_query2(plan.l_xyz[li + 1], plan.l_xyz[li], radii, nsamples))   # both radii, one pass
        self._m("ball")
        for i in range(3, -1, -1):
            d2, nn_idx = _ext.three_nn(plan.l_xyz[i], plan.l_xyz[i + 1])
            plan.nn[i] = (nn_idx, three_nn_weights(d2))
        self._m("three_nn")
        return plan

    def geometry(self, pointcloud: torch.Tensor, fps_chunk: int = 0) -> "GeoPlan":
        """everything of the forward pass that depends on the coordinates only"""
        return self.queries(self.sampling(pointcloud, fps_chunk))

    @torch.no_grad()
    def features(self, pointcloud: torch.Tensor, plan: "GeoPlan", reserve_sms: int = 0, reserve_levels: int = 5,
                 out_rows: torch.Tensor | None = None, col0: int = 0) -> torch.Tensor:
        """The shared MLPs of all SA / FP levels on a geometry plan -> [B,128,N].  reserve_sms: SMs the persistent
        MLP kernels leave free for kernels of other streams (the next batch's sampling); reserve_levels: the SA levels
        0 .. reserve_levels-1 do so (5: the FP modules too) -- the sampling of the next batch is over well before the
        MLPs are, and the later layers then take the whole machine.
        out_rows [B*N, ldo]: FP1 writes the features TF32-rounded and point-major into its columns col0 .. col0+127
        instead (the DenseFusion table of FusedPVN3D), and out_rows is returned."""
        b, _, width = pointcloud.shape
        c0 = width - 3
        rs_all = int(reserve_sms)
        if not plan.ball:
            self.queries(plan)
        # level-0 descriptors are columns 3.. of the input rows themselves (point-major already)
        feats: List[Tuple[int, int, int]] = [(pointcloud.data_ptr() + 12, width, c0)]   # (address, ld, channels)
        l_feat = [pointcloud]          # l_feat[i]: tensor owning level i's descriptors (point-major)
        l_xyz = plan.l_xyz
        table0 = None
        for li, (npoint, radii, nsamples, _) in enumerate(SA_SPEC):
            rs = rs_all if li < reserve_levels else 0
            x, new_xyz = l_xyz[li], l_xyz[li + 1]
            fptr, ldf, c_feat = feats[-1]
            out_l = torch.empty((b, npoint, self.sa_out[li]), dtype=torch.float32, device=self.dev)
            table = sa_factor_table(x, fptr, ldf, c_feat, self.sa_fact[li][0][0].k_pad)   # shared by both scales
            if li == 0:
                table0 = table                                                          # FP1's skip columns
            col = 0
            for idx, (first, wx, b1), (l2, l3, fused) in zip(plan.ball[li], self.sa_fact[li], self.sa[li]):
                u = mlp_dense(table, first, relu=False, a_tf32=True, reserve=rs)        # once per point
                v = sa_centre_term(new_xyz, wx, b1)                                     # once per centre
                # the level tables of SA1-3 are stored TF32-rounded, as their readers (the next level's factor table,
                # the skip columns of FP2-4) round them anyway; SA4's feeds the fp32 interpolation of FP4
                fused(u, v, idx, x.size(1), l2, l3, out=out_l.view(b * npoint, -1), col0=col, round_out=li < 3,
                      reserve=rs)
                col += l3.n
            self._m("mlp")
            feats.append((out_l.data_ptr(), out_l.size(-1), out_l.size(-1)))
            l_feat.append(out_l)
        # feature propagation, deepest first (pvn3d.py:149-152)
        rs = rs_all if reserve_levels >= 5 else 0
        for i in range(3, 0, -1):
            unknown, known = l_xyz[i], l_xyz[i + 1]
            nn_idx, nn_w = plan.nn[i]
            sptr, lds, c1 = feats[i]
            l1, l2 = self.fp[i]
            h = mlp_fp2(l_feat[i + 1], nn_idx, nn_w, sptr, lds, c1, l1, l2, reserve=rs)   # level tables stay full fp32
            l_feat[i] = h.view(b, unknown.size(1), -1)
            self._m("mlp")
        # FP1, factored -- it pays only where the known descriptors are much wider than the layer and the skip is
        # narrow: 256 + 6 -> 128 at 12288 points (DESIGN.md section 4)
        lk, ls, l2 = self.fp1
        nn_idx, nn_w = plan.nn[0]
        kf2d = l_feat[1].reshape(-1, l_feat[1].size(-1))
        assert kf2d.size(-1) == lk.k
        pk = mlp_dense(kf2d, lk, relu=False, reserve=rs)                                   # once per known point
        # S = W1s . table0 + b1 stays on chip; the module's output IS the network's, written channel-major ([B,128,N])
        # or into the caller's row table
        if out_rows is not None:
            mlp_fp_fact2_rows(pk, table0, nn_idx, nn_w, l_xyz[1].size(1), ls, l2, out_rows, col0, reserve=rs)
            self._m("mlp")
            return out_rows
        h = mlp_fp_fact2(pk, table0, nn_idx, nn_w, l_xyz[1].size(1), ls, l2, reserve=rs)
        self._m("mlp")
        return h if l2.n == l2.n_pad else h[:, :l2.n].contiguous()

    @torch.no_grad()
    def forward(self, pointcloud: torch.Tensor, out_rows: torch.Tensor | None = None, col0: int = 0) -> torch.Tensor:
        """pointcloud [B,N,3+C] f32 contiguous on device -> features [B,128,N] (as the reference returns), or written
        into columns col0 .. col0+127 of out_rows [B*N, ldo] (see features)"""
        return self.features(pointcloud, self.geometry(pointcloud), out_rows=out_rows, col0=col0)

    __call__ = forward
