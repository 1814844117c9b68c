"""DenseFusion + the three per-point heads of PVN3D on the tensor-core layer kernel (SURVEY section 8 f3).

Reference: pvn3d/lib/pvn3d.py:157-182 (DenseFusion), :245-267 (SEG_layer / KpOF_layer / CtrOf_layer: Conv1d 1x1 + BN1d +
ReLU stacks on the 1792-channel fused feature), :297-308 (output layouts).  198 GFLOP per 12288-point frame of 1x1
convolutions -- 11x the PointNet++ shared MLPs -- and what `demo.py` waits on once hot paths A and B are fast.

    heads = FusedHeads(model.rgbd_feat, model.SEG_layer, model.KpOF_layer, model.CtrOf_layer)
    pred_kp_of, pred_rgbd_seg, pred_ctr_of = heads(rgb_emb, pcld_emb)       # as PVN3D.forward returns them

Everything runs point-major ([B*N, C] rows) through `pvn3d_mlp_dense*` (wgmma tf32, weights by TMA):
  * conv2_rgb, conv2_cld and conv3 read the same 256 columns [rgb | cld]: ONE launch with a block-structured
    [1024 x 256] weight writes feat_2 and conv3's output next to feat_1 in one activation table;
  * conv4 (512 -> 1024) is only ever averaged over the points (AvgPool1d, :165,178): its epilogue sums relu(.) over
    32-row groups (`pvn3d_mlp_dense_sum32`) instead of storing 1.6 GB of activations per 32-frame batch;
  * the pooled feature is a per-FRAME constant broadcast to every point (:180-182), so the 1024 columns it occupies in
    each head's first layer (57 % of that layer's K) fold into a per-frame bias W_ap . g_b + b
    (`pvn3d_mlp_dense_frame_bias`): K = 768 instead of 1792.
Precision: TF32 operands, fp32 accumulation -- the class of the reference's default cuDNN convolutions; the per-frame
bias and the mean are fp32/fp64.  Host glue (packing [rgb | cld] rows, output permutes) uses torch copies.
"""
from __future__ import annotations

from typing import List, Tuple

import torch

from . import _ext, _lib
from ._lib import check, ptr
from .mlp import PackedLayer, _flags, _stream, fold_conv_bn, tf32_round


def _conv1d_wb(conv: torch.nn.Conv1d) -> Tuple[torch.Tensor, torch.Tensor]:
    w = conv.weight.detach().float().flatten(1)
    b = conv.bias.detach().float() if conv.bias is not None else torch.zeros(w.size(0), device=w.device)
    return w, b


def _dense(a_ptr: int, lda: int, a_cols: int, rows: int, layer: PackedLayer, out: torch.Tensor, col0: int = 0, relu=True,
           round_out=True, a_tf32=True):
    lib = _lib.load()
    dev = out.device
    with torch.cuda.device(dev):
        rc = lib.pvn3d_mlp_dense(a_ptr, lda, a_cols, rows, ptr(layer.w), ptr(layer.bias), layer.k_pad, layer.n_pad,
                                 _flags(relu, round_out, a_tf32), 0, ptr(out), out.size(-1), col0, _stream(dev))
    check(rc, "pvn3d_mlp_dense")
    return out


class _Head:
    """one Conv1d stack: first layer split into [feat_1 | feat_2] columns + the pooled-feature columns"""

    def __init__(self, seq: torch.nn.Module, dev):
        blocks = list(seq.children())
        w1, b1 = fold_conv_bn(blocks[0])                      # [1024, 1792]
        self.first = PackedLayer(w1[:, :768].contiguous(), torch.zeros_like(b1))
        self.w_ap = w1[:, 768:].double().to(dev)               # columns of the broadcast global feature
        self.b1 = b1.double().to(dev)
        self.rest: List[PackedLayer] = []
        prev = self.first.n_pad
        for blk in blocks[1:]:
            w, b = fold_conv_bn(blk)
            pl = PackedLayer(w, b, prev)
            prev = pl.n_pad
            self.rest.append(pl)
        self.n_out = self.rest[-1].n
        self.relu_last = hasattr(blocks[-1], "activation")


class FusedHeads:
    def __init__(self, rgbd_feat: torch.nn.Module, seg_layer: torch.nn.Module, kpof_layer: torch.nn.Module,
                 ctrof_layer: torch.nn.Module, device="cuda"):
        self.dev = torch.device(device)
        if self.dev.type != "cuda":
            raise RuntimeError("FusedHeads: CUDA only -- no CPU fallback")
        rgbd_feat, seg_layer, kpof_layer, ctrof_layer = (m.to(self.dev).eval() for m in (rgbd_feat, seg_layer, kpof_layer, ctrof_layer))
        w2r, b2r = _conv1d_wb(rgbd_feat.conv2_rgb)             # 128 -> 256 on rgb
        w2c, b2c = _conv1d_wb(rgbd_feat.conv2_cld)             # 128 -> 256 on cld
        w3, b3 = _conv1d_wb(rgbd_feat.conv3)                   # 256 -> 512 on [rgb | cld]
        w4, b4 = _conv1d_wb(rgbd_feat.conv4)                   # 512 -> 1024
        z = torch.zeros_like(w2r)
        wa = torch.cat([torch.cat([w2r, z], 1), torch.cat([z, w2c], 1), w3], 0)     # [1024, 256]: feat_2 (512) | conv3 (512)
        self.la = PackedLayer(wa, torch.cat([b2r, b2c, b3]))
        self.lb = PackedLayer(w4, b4, 512)
        self.heads = [_Head(s, self.dev) for s in (seg_layer, kpof_layer, ctrof_layer)]

    #: columns of the activation table: [feat_1 = rgb (128) | cld (128)] [feat_2 (512)] [conv3 output (512)]
    TABLE_COLS = 1280
    RGB_COL0, CLD_COL0 = 0, 128

    def new_table(self, rows: int) -> torch.Tensor:
        """an uninitialised activation table for `rows` = B*N points; run() expects its columns RGB_COL0 .. +127 and
        CLD_COL0 .. +127 filled with the TF32-rounded point-major embeddings"""
        return torch.empty((rows, self.TABLE_COLS), dtype=torch.float32, device=self.dev)

    @torch.no_grad()
    def forward(self, rgb_emb: torch.Tensor, cld_emb: torch.Tensor):
        """rgb_emb [B,128,N] (the CNN embedding gathered at the sampled pixels, pvn3d.py:291-293), cld_emb [B,128,N]
        (Pointnet2MSG.forward) -> (pred_kp_of [B,K,N,3], pred_rgbd_seg [B,N,n_cls], pred_ctr_of [B,1,N,3])"""
        assert rgb_emb.is_cuda and cld_emb.is_cuda and rgb_emb.shape == cld_emb.shape and rgb_emb.size(1) == 128
        b, _, n = cld_emb.shape
        rows = b * n
        x = self.new_table(rows)
        x[:, :128] = tf32_round(_ext.transpose_cn_to_nc(rgb_emb.contiguous().float())).view(rows, 128)
        x[:, 128:256] = tf32_round(_ext.transpose_cn_to_nc(cld_emb.contiguous().float())).view(rows, 128)
        return self.run(x, b, n)

    @torch.no_grad()
    def run(self, x: torch.Tensor, b: int, n: int):
        """DenseFusion and the heads on an activation table x [B*N, TABLE_COLS] (new_table) whose first 256 columns
        hold feat_1 -> the outputs of forward().  Columns 256.. are overwritten."""
        assert x.shape == (b * n, self.TABLE_COLS) and x.is_contiguous() and x.is_cuda
        lib = _lib.load()
        rows = b * n
        _dense(x.data_ptr(), 1280, 256, rows, self.la, x, col0=256)                      # feat_2 and relu(conv3(feat_1))
        # mean over the points of relu(conv4(.)): 32-row partial sums straight from the accumulator
        groups = (rows + 31) // 32
        part = torch.empty((groups, self.lb.n_pad), dtype=torch.float32, device=self.dev)
        with torch.cuda.device(self.dev):
            rc = lib.pvn3d_mlp_dense_sum32(x.data_ptr() + 768 * 4, 1280, 512, rows, ptr(self.lb.w), ptr(self.lb.bias),
                                           self.lb.k_pad, self.lb.n_pad, _flags(True, a_tf32=True), ptr(part), part.size(-1), 0,
                                           _stream(self.dev))
        check(rc, "pvn3d_mlp_dense_sum32")
        if n % 32 == 0:
            ap = part.view(b, n // 32, -1).double().sum(1) / n                           # [B, 1024] AvgPool1d(num_points)
        else:   # 32-row groups straddle frames: per-point activations through the plain layer, then the mean
            full = torch.empty((rows, self.lb.n_pad), dtype=torch.float32, device=self.dev)
            _dense(x.data_ptr() + 768 * 4, 1280, 512, rows, self.lb, full, round_out=False)
            ap = full.view(b, n, -1).double().mean(1)
        outs = []
        for hd in self.heads:
            fb = (ap[:, : hd.w_ap.size(1)] @ hd.w_ap.t() + hd.b1).float()                # per-frame bias [B, 1024]
            fbp = torch.zeros((b, hd.first.n_pad), dtype=torch.float32, device=self.dev)
            fbp[:, : fb.size(1)] = fb
            h = torch.empty((rows, hd.first.n_pad), dtype=torch.float32, device=self.dev)
            if n % 128 == 0:
                with torch.cuda.device(self.dev):
                    rc = lib.pvn3d_mlp_dense_frame_bias(x.data_ptr(), 1280, 768, rows, n, ptr(hd.first.w), ptr(fbp), hd.first.k_pad,
                                                        hd.first.n_pad, _flags(True, True, True), ptr(h), h.size(-1), 0,
                                                        _stream(self.dev))
                check(rc, "pvn3d_mlp_dense_frame_bias")
            else:       # a 128-row tile may straddle frames: one launch per frame with that frame's bias
                for bi in range(b):
                    layer = PackedLayer.__new__(PackedLayer)
                    layer.__dict__.update(hd.first.__dict__)
                    layer.bias = fbp[bi].contiguous()
                    _dense(x.data_ptr() + bi * n * 1280 * 4, 1280, 768, n, layer, h[bi * n:(bi + 1) * n])
            for li, pl in enumerate(hd.rest):
                last = li == len(hd.rest) - 1
                nxt = torch.empty((rows, pl.n_pad), dtype=torch.float32, device=self.dev)
                _dense(h.data_ptr(), h.size(-1), h.size(-1), rows, pl, nxt, relu=(not last) or hd.relu_last, round_out=not last)
                h = nxt
            outs.append(h[:, : hd.n_out])
        seg, kp, ctr = outs
        k = kp.size(1) // 3
        pred_rgbd_seg = seg.reshape(b, n, -1).contiguous()                                # .transpose(1, 2) of [B,n_cls,N] (:297)
        pred_kp_of = kp.reshape(b, n, k, 3).permute(0, 2, 1, 3).contiguous()              # [B,K,N,3] (:298-302)
        pred_ctr_of = ctr.reshape(b, n, 1, 3).permute(0, 2, 1, 3).contiguous()            # [B,1,N,3] (:303-306)
        return pred_kp_of, pred_rgbd_seg, pred_ctr_of

    __call__ = forward


def reference_layout_modules(n_classes: int = 22, n_kps: int = 8):
    """random-init DenseFusion + head stacks with the reference's module structure (pvn3d.py:157-182,245-267):
    Conv1d(1x1) [+ BatchNorm1d] [+ ReLU] blocks named conv / normlayer.bn / activation, so that a reference
    checkpoint's `rgbd_feat.*`, `SEG_layer.*`, `KpOF_layer.*`, `CtrOf_layer.*` entries load unchanged.  For bench.py
    and for callers without the reference tree."""
    nn = torch.nn

    class DenseFusion(nn.Module):
        def __init__(self):
            super().__init__()
            self.conv2_rgb = nn.Conv1d(128, 256, 1)
            self.conv2_cld = nn.Conv1d(128, 256, 1)
            self.conv3 = nn.Conv1d(256, 512, 1)
            self.conv4 = nn.Conv1d(512, 1024, 1)

    def block(c_in, c_out, bn, act):
        blk = nn.Sequential()
        blk.add_module("conv", nn.Conv1d(c_in, c_out, 1, bias=not bn))
        if bn:
            norm = nn.Sequential()
            norm.add_module("bn", nn.BatchNorm1d(c_out))
            blk.add_module("normlayer", norm)
        if act:
            blk.add_module("activation", nn.ReLU(inplace=True))
        return blk

    def stack(widths, out):
        seq = nn.Sequential()
        c = 1792
        for i, w in enumerate(widths):
            seq.add_module(str(i), block(c, w, True, True))
            c = w
        seq.add_module(str(len(widths)), block(c, out, False, False))
        return seq

    return DenseFusion(), stack((1024, 512, 128), n_classes), stack((1024, 512, 256), n_kps * 3), stack((1024, 512, 128), 3)
