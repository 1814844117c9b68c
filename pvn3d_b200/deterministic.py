"""Deterministic backward for PSPNet's adaptive average pooling and bilinear upsampling.

torch has no deterministic CUDA backward for either op: under torch.use_deterministic_algorithms(True) the reference's
`lib/pspnet.py` (nn.AdaptiveAvgPool2d, F.upsample(..., mode='bilinear'), nn.Upsample(scale_factor=2,
mode='bilinear', align_corners=True)) raises at its first backward.  The autograd functions here run torch's own
forward, so forward bits never change, and a backward that depends on the mode:
  * deterministic mode on (warn_only included), a float32 CUDA NCHW gradient: pvn3d_adaptive_avg_pool2d_backward /
    pvn3d_upsample_bilinear2d_backward (csrc/determinism.cu), which write every input-gradient element once, summing
    its contributions in ascending output order;
  * otherwise torch's own backward op, as if the module had never been wrapped.

`compat.install(..., patch_deterministic=True)` routes the reference's PSPModule and PSPUpsample through them.
"""
from __future__ import annotations

import types

import torch
import torch.nn.functional as F
from torch import nn

from ._lib import call, ptr


def _ordered(g: torch.Tensor) -> bool:
    return (torch.are_deterministic_algorithms_enabled() and g.is_cuda and g.dtype == torch.float32
            and g.dim() == 4)


def _pair(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


class _AdaptiveAvgPool2d(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, output_size):
        ctx.save_for_backward(x)
        return F.adaptive_avg_pool2d(x, output_size)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        if not _ordered(g):
            return torch.ops.aten._adaptive_avg_pool2d_backward(g, x), None
        g = g.contiguous()
        n, c, oh, ow = g.shape
        ih, iw = x.shape[-2:]
        out = torch.empty((n, c, ih, iw), dtype=g.dtype, device=g.device)
        call("pvn3d_adaptive_avg_pool2d_backward", g.device, ptr(g), n * c, ih, iw, oh, ow, ptr(out))
        return out, None


class _UpsampleBilinear2d(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, size, scale_factor, align_corners):
        out = F.interpolate(x, size=size, scale_factor=scale_factor, mode="bilinear", align_corners=align_corners)
        # the scales torch's op receives: interpolate passes a scale factor through (recompute_scale_factor unset)
        ctx.scales = _pair(scale_factor) if scale_factor is not None else (None, None)
        ctx.in_size, ctx.align = tuple(x.shape), align_corners
        return out

    @staticmethod
    def backward(ctx, g):
        oh, ow = g.shape[-2:]
        sh, sw = ctx.scales
        if not _ordered(g):
            gi = torch.ops.aten.upsample_bilinear2d_backward(g, [oh, ow], list(ctx.in_size), ctx.align, sh, sw)
            return gi, None, None, None
        g = g.contiguous()
        n, c, ih, iw = ctx.in_size
        out = torch.empty(ctx.in_size, dtype=g.dtype, device=g.device)
        call("pvn3d_upsample_bilinear2d_backward", g.device, ptr(g), n * c, ih, iw, oh, ow, int(ctx.align),
             float(sh or 0.0), float(sw or 0.0), ptr(out))
        return out, None, None, None


def adaptive_avg_pool2d(x: torch.Tensor, output_size) -> torch.Tensor:
    """F.adaptive_avg_pool2d with the deterministic backward (4-D inputs; others run torch's op).  A 1x1 output runs
    torch's op as is: torch computes it as a mean, whose backward is already deterministic and never refused."""
    oh, ow = (x.size(d) if o is None else int(o) for d, o in zip((-2, -1), _pair(output_size)))
    if x.dim() != 4 or (oh, ow) == (1, 1):
        return F.adaptive_avg_pool2d(x, output_size)
    return _AdaptiveAvgPool2d.apply(x, output_size)


def interpolate(input, size=None, scale_factor=None, mode="nearest", align_corners=None, recompute_scale_factor=None,
                antialias=False):
    """F.interpolate; 4-D bilinear calls (without antialias or recompute_scale_factor) get the deterministic
    backward, everything else runs torch's op"""
    if mode == "bilinear" and input.dim() == 4 and not antialias and not recompute_scale_factor:
        if isinstance(scale_factor, list):
            scale_factor = tuple(scale_factor)
        if isinstance(size, list):
            size = tuple(size)
        return _UpsampleBilinear2d.apply(input, size, scale_factor, bool(align_corners))
    return F.interpolate(input, size, scale_factor, mode, align_corners, recompute_scale_factor, antialias)


def upsample(input, size=None, scale_factor=None, mode="nearest", align_corners=None):
    """F.upsample (the deprecated spelling lib/pspnet.py uses) on `interpolate`"""
    return interpolate(input, size, scale_factor, mode, align_corners)


class AdaptiveAvgPool2d(nn.AdaptiveAvgPool2d):
    """nn.AdaptiveAvgPool2d with the deterministic backward"""

    def forward(self, x):
        return adaptive_avg_pool2d(x, self.output_size)


class Upsample(nn.Upsample):
    """nn.Upsample with the deterministic bilinear backward"""

    def forward(self, x):
        return interpolate(x, self.size, self.scale_factor, self.mode, self.align_corners,
                           recompute_scale_factor=self.recompute_scale_factor)


def adopt(module: nn.Module) -> None:
    """Give every plain nn.AdaptiveAvgPool2d / nn.Upsample under `module` the deterministic backward, in place (the
    instance's class becomes the subclass above; parameters, buffers and state dicts are untouched)."""
    for m in module.modules():
        if type(m) is nn.AdaptiveAvgPool2d:
            m.__class__ = AdaptiveAvgPool2d
        elif type(m) is nn.Upsample:
            m.__class__ = Upsample


def functional() -> types.ModuleType:
    """torch.nn.functional with `upsample` and `interpolate` replaced by this module's"""
    mod = types.ModuleType("pvn3d_b200.deterministic.functional")
    mod.__getattr__ = lambda name: getattr(F, name)
    mod.upsample, mod.interpolate, mod.adaptive_avg_pool2d = upsample, interpolate, adaptive_avg_pool2d
    return mod
