"""Inputs shared by the CNN-tail tests (test infrastructure, no conftest): half-resolution maps and `choose` indices
that hit every border case of the 3x3 taps."""
import torch

# (h, w) of the half-resolution map: the smallest useful image, odd half sizes, and the dataset size
SIZES = [(4, 5), (30, 41), (240, 320)]


def half_map(b, h, w, seed=0, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(b, 64, h, w, generator=g, dtype=torch.float64).to(dtype)


def border_choose(b, n, hh, ww, seed=0):
    """[b,1,n] int64: in every frame the four corners, a pixel of every edge, the pixels next to them, random interior
    pixels and repeats"""
    g = torch.Generator().manual_seed(seed)
    fixed = [0, ww - 1, (hh - 1) * ww, hh * ww - 1,                       # corners
             ww // 2, (hh - 1) * ww + ww // 2, (hh // 2) * ww, (hh // 2) * ww + ww - 1,   # edges
             ww + 1, 2 * ww - 2, (hh - 2) * ww + 1, (hh - 1) * ww - 2,     # one pixel inside the corners
             0, hh * ww - 1]                                                # repeats
    out = torch.empty((b, 1, n), dtype=torch.int64)
    for f in range(b):
        rnd = torch.randint(0, hh * ww, (max(n - len(fixed), 0),), generator=g)
        row = torch.cat([torch.tensor(fixed, dtype=torch.int64), rnd])[:n]
        out[f, 0] = row[torch.randperm(n, generator=g)]
    return out
