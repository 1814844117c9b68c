"""The whole PVN3D network forward (reference pvn3d/lib/pvn3d.py:269-310) on the library's engines: FusedPVN3D.

    net = FusedPVN3D(model, "cuda")                     # model: a reference PVN3D, or any module with its attributes
    pred_kp_of, pred_rgbd_seg, pred_ctr_of = net(pointcloud, rgb, choose)     # as PVN3D.forward returns them

One call, device resident, in the reference's order:
  1. model.cnn(rgb) unchanged (stock PyTorch / cuDNN);
  2. the embedding at the sampled pixels -> columns 0..127 of the DenseFusion activation table (pvn3d_gather_pixel_rows:
     no [B,128,N] int64 index, no transpose, no copy);
  3. FusedPointnet2MSG, whose last launch (FP1, pvn3d_mlp_fp_fact2_rows) writes columns 128..255 of the same table;
  4. the rest of FusedHeads on that table.
The outputs are bit-identical to FusedHeads(gathered rgb_emb, FusedPointnet2MSG(pointcloud)).

Divergence from the reference: a `choose` index outside [0, H*W) gives that point a row of NaN (and NaN outputs)
where torch.gather would raise.
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import check, ptr
from .heads import FusedHeads
from .mlp import FusedPointnet2MSG, _stream


def gather_pixel_rows(emb: torch.Tensor, choose: torch.Tensor, out: torch.Tensor, col0: int = 0) -> torch.Tensor:
    """emb [B,C,H,W] or [B,C,H*W] f32, choose [B,1,N] int64 -> out[b*N + p, col0 + c] = tf32(emb[b, c, choose[b,0,p]])
    (pvn3d_gather_pixel_rows): the rows of tf32_round(torch.gather(emb.view(B,C,-1), 2, choose.repeat(1,C,1)).transpose(1,
    2)), bit for bit.  An index outside [0, H*W) writes a row of NaN."""
    b, c = emb.size(0), emb.size(1)
    emb = emb.reshape(b, c, -1)
    if emb.dtype != torch.float32 or not emb.is_contiguous():
        raise ValueError("gather_pixel_rows: emb must be a contiguous float32 tensor")
    if choose.dtype != torch.int64 or choose.dim() != 3 or choose.size(0) != b or choose.size(1) != 1:
        raise ValueError(f"gather_pixel_rows: choose must be int64 [B,1,N], got {choose.dtype} {tuple(choose.shape)}")
    choose = choose.contiguous()
    n = choose.size(2)
    if out.dim() != 2 or out.size(0) != b * n or out.stride(1) != 1:
        raise ValueError(f"gather_pixel_rows: out must be rows [B*N, ldo], got {tuple(out.shape)}")
    lib = _lib.load()
    with torch.cuda.device(emb.device):
        rc = lib.pvn3d_gather_pixel_rows(ptr(emb), b, c, emb.size(2), ptr(choose), n, ptr(out), out.stride(0), col0,
                                         _stream(emb.device))
    check(rc, "pvn3d_gather_pixel_rows")
    return out


class FusedPVN3D:
    """Inference engine for PVN3D.forward (see module docstring).  `model` provides cnn, pointnet2, rgbd_feat,
    SEG_layer, KpOF_layer, CtrOf_layer and num_kps; the weights are folded at construction (a later change to them
    needs a new engine)."""

    def __init__(self, model: torch.nn.Module, device="cuda"):
        self.dev = torch.device(device)
        if self.dev.type != "cuda":
            raise RuntimeError("FusedPVN3D: CUDA only -- no CPU fallback")
        self.cnn = model.cnn
        self.num_kps = int(model.num_kps)
        ap1 = getattr(model.rgbd_feat, "ap1", None)
        ks = None if ap1 is None else ap1.kernel_size
        self.num_points = None if ks is None else int(ks[0] if isinstance(ks, (tuple, list)) else ks)
        self.pointnet2 = FusedPointnet2MSG(model.pointnet2, self.dev)
        self.heads = FusedHeads(model.rgbd_feat, model.SEG_layer, model.KpOF_layer, model.CtrOf_layer, self.dev)

    @torch.no_grad()
    def forward(self, pointcloud: torch.Tensor, rgb: torch.Tensor, choose: torch.Tensor):
        """pointcloud [B,N,3+C] f32, rgb [B,3,H,W], choose [B,1,N] int64, all on the device ->
        (pred_kp_of [B,K,N,3], pred_rgbd_seg [B,N,n_cls], pred_ctr_of [B,1,N,3])"""
        b, n = pointcloud.size(0), pointcloud.size(1)
        if self.num_points is not None and n != self.num_points:
            # the reference fails here too: DenseFusion's AvgPool1d(num_points) does not pool N points to one
            raise ValueError(f"FusedPVN3D: {n} points, but rgbd_feat.ap1 pools over num_points = {self.num_points}")
        out_rgb, _ = self.cnn(rgb)
        if out_rgb.size(0) != b or out_rgb.size(1) != 128:
            raise ValueError(f"FusedPVN3D: the CNN embedding is {tuple(out_rgb.shape)}, expected [{b}, 128, H, W]")
        x = self.heads.new_table(b * n)
        gather_pixel_rows(out_rgb.float().contiguous(), choose, x, col0=FusedHeads.RGB_COL0)
        self.pointnet2(pointcloud.float().contiguous(), out_rows=x, col0=FusedHeads.CLD_COL0)
        kp, seg, ctr = self.heads.run(x, b, n)
        assert kp.size(1) == self.num_kps
        return kp, seg, ctr

    __call__ = forward
