"""The full-resolution tail of PVN3D's CNN, evaluated only at the sampled pixels: PspTail.

The reference's CNN (Modified_PSPNet, pspnet.py:48-90) ends with

    p   = up_3(p)        # bilinear x2 (align_corners) -> Conv2d(64,64,3,padding 1) -> BatchNorm2d -> PReLU, at H x W
    emb = final(p)       # Conv2d(64,128,1) at H x W

and PVN3D.forward keeps N of the H*W columns of emb (pvn3d.py:288-292).  Every step is per pixel with a 3x3 receptive
field in the up-sampled map, so the kept columns can be computed alone: PspTail folds up_3's conv + BN and `final` into
two layers of pvn3d_psp_tail_rows (576 -> 64, PReLU, 64 -> 128), runs the CNN up to up_2 on the model's own modules
(`trunk`) and writes the rows straight into the heads' activation table (`rows`).  up_3, final and final_seg never run.

    tail = PspTail.from_cnn(model.cnn)       # None unless the CNN has the reference's layout
    tail.rows(tail.trunk(rgb), choose, table, col0)
"""
from __future__ import annotations

import ctypes

import torch

from ._lib import call, ptr
from .mlp import PackedLayer, _layer_struct

_ATTRS = ("feats", "psp", "drop_1", "up_1", "up_2", "up_3", "drop_2", "final")
C_MID, C_EMB = 64, 128


def _pair(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


def _is_conv(m, c_in, c_out, k, pad) -> bool:
    return (isinstance(m, torch.nn.Conv2d) and m.in_channels == c_in and m.out_channels == c_out
            and _pair(m.kernel_size) == (k, k) and _pair(m.stride) == (1, 1) and _pair(m.padding) == (pad, pad)
            and _pair(m.dilation) == (1, 1) and m.groups == 1 and m.padding_mode == "zeros")


def fold_tail(model: torch.nn.Module, dtype=torch.float32):
    """(w1 [64, 576], b1 [64], slope [64], w2 [128, 64], b2 [128]) in `dtype`, folded in float64, from a
    model with the reference's tail, BN in eval mode folded by attribute (BatchNorm2d or its SyncBatchNorm conversion); None for any other layout.
    w1[o, (3 ky + kx) * 64 + c] = gamma_o / sqrt(var_o + eps) * conv.weight[o, c, ky, kx]."""
    if not all(hasattr(model, a) for a in _ATTRS):
        return None
    seq, final = getattr(model.up_3, "conv", None), model.final
    if not (isinstance(seq, torch.nn.Sequential) and len(seq) == 4 and isinstance(final, torch.nn.Sequential) and len(final) == 1):
        return None
    up, conv, bn, act = seq
    if not (isinstance(up, torch.nn.Upsample) and up.mode == "bilinear" and up.align_corners is True and up.size is None
            and up.scale_factor is not None and tuple(float(s) for s in _pair(up.scale_factor)) == (2.0, 2.0)):
        return None
    if not (_is_conv(conv, C_MID, C_MID, 3, 1) and _is_conv(final[0], C_MID, C_EMB, 1, 0)):
        return None
    stats = [getattr(bn, a, None) for a in ("weight", "bias", "running_mean", "running_var")]
    if any(not isinstance(t, torch.Tensor) or t.numel() != C_MID for t in stats) or not hasattr(bn, "eps"):
        return None
    if not (isinstance(act, torch.nn.PReLU) and act.weight.numel() in (1, C_MID)):
        return None
    gamma, beta, mean, var = (t.detach().double() for t in stats)
    scale = gamma / torch.sqrt(var + bn.eps)
    w = conv.weight.detach().double() * scale[:, None, None, None]            # [o, c, ky, kx]
    w1 = w.permute(0, 2, 3, 1).reshape(C_MID, 9 * C_MID)                       # k = (3 ky + kx) * 64 + c
    cb = conv.bias.detach().double() if conv.bias is not None else torch.zeros_like(mean)
    b1 = (cb - mean) * scale + beta
    slope = act.weight.detach().double().expand(C_MID)
    w2 = final[0].weight.detach().double().reshape(C_EMB, C_MID)
    b2 = final[0].bias.detach().double() if final[0].bias is not None else torch.zeros(C_EMB, dtype=torch.float64, device=w2.device)
    return tuple(t.to(dtype).contiguous() for t in (w1, b1, slope, w2, b2))


class PspTail:
    """The folded tail of one CNN (see module docstring).  The weights are folded at construction; a later change to
    them needs a new PspTail."""

    def __init__(self, model: torch.nn.Module, folded, device):
        self.model = model
        w1, b1, slope, w2, b2 = (t.to(device) for t in folded)
        self.layer1 = PackedLayer(w1, b1)
        self.layer2 = PackedLayer(w2, b2)
        self.slope = slope.contiguous()

    @classmethod
    def from_cnn(cls, cnn: torch.nn.Module, device=None) -> "PspTail | None":
        """the tail of `cnn` (a Modified_PSPNet, or a wrapper holding one as `.model`) on `device` (default: where its
        weights are), or None when the CNN does not have that layout"""
        model = cnn.model if hasattr(cnn, "model") else cnn
        folded = fold_tail(model)
        if folded is None:
            return None
        return cls(model, folded, folded[0].device if device is None else device)

    def trunk(self, rgb: torch.Tensor) -> torch.Tensor:
        """Modified_PSPNet.forward up to the input of up_3 (pspnet.py:78-86) on the model's own modules ->
        [B, 64, H/2, W/2]"""
        m = self.model
        f, _ = m.feats(rgb)
        p = m.drop_1(m.psp(f))
        p = m.drop_2(m.up_1(p))
        return m.drop_2(m.up_2(p))

    def rows(self, x_half: torch.Tensor, choose: torch.Tensor, out: torch.Tensor, col0: int = 0) -> torch.Tensor:
        """x_half [B,64,h,w] f32 (or bf16 from an autocast CNN), choose [B,1,N] int64 indices into the 2h x 2w image ->
        out[b*N + p, col0 : col0+128] = final(up_3(x_half))[b, :, choose[b,0,p]] to TF32 accuracy (pvn3d_psp_tail_rows;
        a bfloat16 `out` takes the rows rounded to bf16, pvn3d_psp_tail_rows_bf16).  An index outside the image writes
        a row of NaN."""
        if x_half.dim() != 4 or x_half.size(1) != C_MID or x_half.dtype not in (torch.float32, torch.bfloat16):
            raise ValueError(f"PspTail.rows: x_half must be f32 or bf16 [B, {C_MID}, h, w], got {x_half.dtype} {tuple(x_half.shape)}")
        b, _, h, w = x_half.shape
        if choose.dtype != torch.int64 or choose.dim() != 3 or choose.size(0) != b or choose.size(1) != 1:
            raise ValueError(f"PspTail.rows: choose must be int64 [B,1,N], got {choose.dtype} {tuple(choose.shape)}")
        choose = choose.contiguous()
        n = choose.size(2)
        if out.dim() != 2 or out.size(0) != b * n or out.stride(1) != 1 or out.dtype not in (torch.float32, torch.bfloat16):
            raise ValueError(f"PspTail.rows: out must be f32 or bf16 rows [B*N, ldo], got {out.dtype} {tuple(out.shape)}")
        # channels-last f32 in one copy: [B, h, w, 64]
        x = torch.empty((b, h, w, C_MID), dtype=torch.float32, device=x_half.device).copy_(x_half.permute(0, 2, 3, 1))
        fn = "pvn3d_psp_tail_rows_bf16" if out.dtype == torch.bfloat16 else "pvn3d_psp_tail_rows"
        l1, l2 = _layer_struct(self.layer1), _layer_struct(self.layer2)
        call(fn, x.device, ptr(x), b, h, w, ptr(choose), n, ctypes.addressof(l1), ctypes.addressof(l2), ptr(self.slope),
             0, ptr(out), out.stride(0), col0)
        return out


def sampled_tail_reference(x_half: torch.Tensor, choose: torch.Tensor, folded, dtype=torch.float64, taps_round=None):
    """The computation of pvn3d_psp_tail_rows in plain torch (the tests' reference): x_half [B,64,h,w], choose [B,1,N],
    folded = fold_tail(model) -> (rows [B*N, 128], hidden [B*N, 64] after the PReLU, taps [B*N, 576]) in `dtype`.
    taps_round: applied to the taps before layer 1 (the kernel rounds them to TF32); no other rounding is modelled.
    Indices must be inside the image."""
    w1, b1, slope, w2, b2 = (t.to(dtype) for t in folded)
    x = x_half.to(dtype)
    b, c, h, w = x.shape
    hh, ww = 2 * h, 2 * w
    n = choose.size(2)
    idx = choose.reshape(b, n)
    y, xx = idx // ww, idx % ww
    frame = torch.arange(b, device=x.device)[:, None].expand(b, n)
    xl = x.permute(0, 2, 3, 1)                                                 # [B, h, w, C]

    def axis(t, n_src):
        num, den = t * (n_src - 1), 2 * n_src - 1
        i0 = torch.div(num, den, rounding_mode="floor")
        return i0, (i0 + 1).clamp(max=n_src - 1), (num - i0 * den).to(dtype) / den

    taps = []
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            ty, tx = y + dy, xx + dx
            inside = ((ty >= 0) & (ty < hh) & (tx >= 0) & (tx < ww)).to(dtype)[..., None]
            i0, i1, ly = axis(ty.clamp(0, hh - 1), h)
            j0, j1, lx = axis(tx.clamp(0, ww - 1), w)
            ly, lx = ly[..., None], lx[..., None]
            top = (1 - lx) * xl[frame, i0, j0] + lx * xl[frame, i0, j1]
            bot = (1 - lx) * xl[frame, i1, j0] + lx * xl[frame, i1, j1]
            taps.append(((1 - ly) * top + ly * bot) * inside)
    taps = torch.cat(taps, -1).reshape(b * n, 9 * c)
    if taps_round is not None:
        taps = taps_round(taps)
    v = taps @ w1.t() + b1
    hidden = torch.where(v >= 0, v, slope * v)
    return hidden @ w2.t() + b2, hidden, taps
