"""Deterministic helpers shared by tests, golden-vector scripts and bench.py (no oracle imports)."""
from __future__ import annotations

import torch


def randomize_bn_(model: torch.nn.Module, seed: int = 1) -> torch.nn.Module:
    """Give every BatchNorm non-trivial affine + running statistics (a fresh model has mean 0 / var 1,
    which would hide BN-folding mistakes).  Same values for any module with the same BN layout."""
    g = torch.Generator().manual_seed(seed)
    for m in model.modules():
        if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
            c = m.num_features
            with torch.no_grad():
                m.weight.copy_(torch.rand(c, generator=g) + 0.5)
                m.bias.copy_(torch.randn(c, generator=g) * 0.1)
                m.running_mean.copy_(torch.randn(c, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return model


def seeded_pointnet2msg(seed: int = 0, bn_seed: int = 1, input_channels: int = 6):
    """torch.manual_seed(seed); Pointnet2MSG() with default init; randomised BN; eval()."""
    from .pointnet2 import Pointnet2MSG

    torch.manual_seed(seed)
    model = Pointnet2MSG(input_channels=input_channels)
    randomize_bn_(model, bn_seed)
    return model.eval()


class StandInCNN(torch.nn.Module):
    """A small seeded stand-in for PVN3D's ModifiedResnet (whose construction fetches a pretrained checkpoint):
    rgb [B,3,H,W] -> ([B,128,H,W] embedding, [B,2,H,W] seg), the pair PVN3D.forward unpacks (pvn3d.py:286)."""

    def __init__(self, seed: int = 0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.conv = torch.nn.Conv2d(3, 128, 1)
        self.seg = torch.nn.Conv2d(128, 2, 1)
        with torch.no_grad():
            for p in self.parameters():
                p.copy_(torch.randn(p.shape, generator=g) * 0.5)

    def forward(self, rgb):
        emb = torch.relu(self.conv(rgb))
        return emb, self.seg(emb)


class _StandInUp(torch.nn.Module):
    """an up-sampling block in the layout of the reference's PSPUpsample: `.conv` = bilinear x2 (align_corners) ->
    Conv2d 3x3 -> BatchNorm2d -> PReLU"""

    def __init__(self, c_in: int, c_out: int, prelu_params: int = 1):
        super().__init__()
        self.conv = torch.nn.Sequential(torch.nn.Upsample(scale_factor=2, mode="bilinear", align_corners=True),
                                        torch.nn.Conv2d(c_in, c_out, 3, padding=1), torch.nn.BatchNorm2d(c_out),
                                        torch.nn.PReLU(prelu_params))

    def forward(self, x):
        return self.conv(x)


class StandInPSPNet(torch.nn.Module):
    """A small seeded CNN with the attribute names, the tail modules and the forward order of the reference's
    Modified_PSPNet (whose construction fetches a pretrained checkpoint): a cheap 1/8-resolution `feats` and `psp`, then
    up_1, up_2, up_3 (64 -> 64), final (64 -> 128) and final_seg.  rgb [B,3,H,W] (H, W multiples of 8) ->
    ([B,128,H,W] embedding, [B,H,W,n_classes] log-probabilities).  BN statistics randomised, PReLU slopes non-default."""

    def __init__(self, seed: int = 0, prelu_params: int = 1, n_classes: int = 22):
        super().__init__()
        torch.manual_seed(seed)
        self.stem = torch.nn.Conv2d(3, 32, 8, stride=8)
        self.psp = torch.nn.Sequential(torch.nn.Conv2d(32, 32, 1), torch.nn.ReLU())
        self.drop_1 = torch.nn.Dropout2d(p=0.3)
        self.up_1 = _StandInUp(32, 32)
        self.up_2 = _StandInUp(32, 64)
        self.up_3 = _StandInUp(64, 64, prelu_params)
        self.drop_2 = torch.nn.Dropout2d(p=0.15)
        self.final = torch.nn.Sequential(torch.nn.Conv2d(64, 128, 1))
        self.final_seg = torch.nn.Sequential(torch.nn.Conv2d(64, n_classes, 1), torch.nn.LogSoftmax(dim=1))
        randomize_bn_(self, seed + 1)
        with torch.no_grad():
            for m in self.modules():
                if isinstance(m, torch.nn.PReLU):
                    m.weight.copy_(torch.rand(m.weight.shape) * 0.4 + 0.05)
        self.eval()

    def feats(self, x):
        f = self.stem(x)
        return f, f.mean((2, 3))

    def forward(self, x):
        f, _ = self.feats(x)
        p = self.drop_1(self.psp(f))
        p = self.drop_2(self.up_1(p))
        p = self.drop_2(self.up_2(p))
        p = self.up_3(p)
        return self.final(p), self.final_seg(p).permute(0, 2, 3, 1).contiguous()


class StandInPVN3D(torch.nn.Module):
    """A module with the attributes of the reference PVN3D (cnn, pointnet2, rgbd_feat, SEG_layer, KpOF_layer,
    CtrOf_layer, num_kps) built from this package's reference-layout modules, and a module-graph forward that computes
    what PVN3D.forward (pvn3d.py:269-310) computes: the unfused, autograd-capable form."""

    def __init__(self, num_points: int, seed: int = 0, n_classes: int = 22, num_kps: int = 8):
        super().__init__()
        from .heads import reference_layout_modules

        self.num_kps = num_kps
        self.cnn = StandInCNN(seed)
        self.pointnet2 = seeded_pointnet2msg(seed, seed + 1)
        torch.manual_seed(seed + 2)
        mods = reference_layout_modules(n_classes, num_kps)
        for i, m in enumerate(mods):
            randomize_bn_(m, seed + 10 + i)
        self.rgbd_feat, self.SEG_layer, self.KpOF_layer, self.CtrOf_layer = mods
        self.rgbd_feat.ap1 = torch.nn.AvgPool1d(num_points)
        self.eval()

    def forward(self, pointcloud, rgb, choose):
        f = torch.nn.functional
        out_rgb, _ = self.cnn(rgb)
        bs, di = out_rgb.shape[:2]
        rgb_emb = torch.gather(out_rgb.view(bs, di, -1), 2, choose.repeat(1, di, 1)).contiguous()
        n = pointcloud.size(1)
        cld_emb = self.pointnet2(pointcloud)
        d = self.rgbd_feat
        feat_1 = torch.cat((rgb_emb, cld_emb), dim=1)
        feat_2 = torch.cat((f.relu(d.conv2_rgb(rgb_emb)), f.relu(d.conv2_cld(cld_emb))), dim=1)
        ap_x = d.ap1(f.relu(d.conv4(f.relu(d.conv3(feat_1))))).view(-1, 1024, 1).repeat(1, 1, n)
        feat = torch.cat([feat_1, feat_2, ap_x], 1)
        seg = self.SEG_layer(feat).transpose(1, 2).contiguous()
        kp = self.KpOF_layer(feat).view(bs, self.num_kps, 3, n).permute(0, 1, 3, 2).contiguous()
        ctr = self.CtrOf_layer(feat).view(bs, 1, 3, n).permute(0, 1, 3, 2).contiguous()
        return kp, seg, ctr


def sample_choose(b: int, n: int, hw: int, seed: int = 0) -> torch.Tensor:
    """[b,1,n] int64 pixel indices as the datasets build them: ascending within a frame; a frame with fewer than n
    candidate pixels repeats them ('wrap' padding).  Frame f draws from min(hw, n * (f + 1) // 2) pixels, so frame 0
    wraps."""
    g = torch.Generator().manual_seed(seed)
    out = torch.empty((b, 1, n), dtype=torch.int64)
    for f in range(b):
        m = min(hw, max(1, n * (f + 1) // 2))
        pick = torch.sort(torch.randperm(hw, generator=g)[:m]).values
        out[f, 0] = pick.repeat((n + m - 1) // m)[:n]
    return out
