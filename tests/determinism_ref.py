"""Float32 restatements of the fixed-order backward contracts (csrc/determinism.cu, include/pvn3d_b200.h), their
float64 adjoints with element-wise bounds, and wrong restatements ("mutants") the checks must reject (test
infrastructure, no conftest).  Everything is torch, on whatever device the operands live on.

Restatements (float32, each element summed from +0.0 one term at a time -- a loop, never a pairwise reduction):
  * ordered_scatter: out[b,c,i] = the terms[b,c,j] with idx[b,j] == i, in ascending j (gather: terms = g; group: g
    flattened over (m, s); interpolate: fl(g[b,c,j] * w[b,j,k]) at slot 3j + k).  Indices outside [0, n) are dropped.
  * pool_backward: grad_in[p,y,x] = the (g[p,oy,ox] / kW) / kH of the bins holding (y, x), in ascending (oy, ox): the
    order of torch's two divisions, pinned against its CUDA backward.
  * upsample_backward: grad_in[p,y,x] = the fl(fl(lh lw) g[p,oy,ox]) of the taps landing on (y, x), in ascending
    output index, within an output in torch's tap order (i1,j1), (i1,j1+j1p), (i1+i1p,j1), (i1+i1p,j1+j1p).

Float64 adjoints: the same linear maps applied exactly (float64 index_add / matrix products), with k = the number of
contributions and S = the sum of their absolute values.  A restatement's error is within (gamma_{k+2} + gamma_k(2^-53))
S: k - 1 additions onto the zero and at most two roundings inside each term (Higham, eq. 3.4 / 4.4).
"""
from __future__ import annotations

import numpy as np
import torch

U32 = 2.0 ** -24
U64 = 2.0 ** -53


def gamma(k, u=U32):
    ku = k.double() * u
    return ku / (1.0 - ku)


# ---- PointNet++ grads -----------------------------------------------------------------------------------------------
def _runs(idx: torch.Tensor, n: int):
    """(key, position, rank) of every in-range entry of idx [B,J], key = b n + idx, grouped by rank (the entry's place
    among the entries of its key, in ascending j)"""
    b, j = idx.shape
    dev = idx.device
    idx = idx.long()
    valid = (idx >= 0) & (idx < n)
    key = (torch.arange(b, device=dev)[:, None] * n + idx)[valid]
    pos = torch.arange(b * j, device=dev).reshape(b, j)[valid]
    order = torch.sort(key, stable=True).indices
    key, pos = key[order], pos[order]
    ar = torch.arange(key.numel(), device=dev)
    first = torch.ones_like(key, dtype=torch.bool)
    first[1:] = key[1:] != key[:-1]
    rank = ar - torch.cummax(torch.where(first, ar, torch.zeros_like(ar)), 0).values
    o2 = torch.sort(rank, stable=True).indices
    return key[o2], pos[o2], rank[o2]


def ordered_scatter(terms: torch.Tensor, idx: torch.Tensor, n: int, order: str = "ascending") -> torch.Tensor:
    """terms [B,C,J] f32, idx [B,J] -> [B,C,n] f32: the sequential float32 sum of each point's terms in ascending j.
    order="descending" is the reversed-order mutant."""
    b, c, j = terms.shape
    key, pos, rank = _runs(idx.reshape(b, j), n)
    if order == "descending":                      # rank counted from the run's end
        cnt = torch.bincount(key, minlength=b * n)
        rank = cnt[key] - 1 - rank
        o = torch.sort(rank, stable=True).indices
        key, pos, rank = key[o], pos[o], rank[o]
    flat = terms.float().permute(1, 0, 2).reshape(c, b * j)
    acc = torch.zeros((c, b * n), dtype=torch.float32, device=terms.device)
    counts = torch.bincount(rank).tolist() if rank.numel() else []
    s = 0
    for cnt in counts:
        ks, ps = key[s:s + cnt], pos[s:s + cnt]   # one term per key at this rank
        acc[:, ks] = acc[:, ks] + flat[:, ps]
        s += cnt
    return acc.reshape(c, b, n).permute(1, 0, 2).contiguous()


def interp_terms32(g: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """g [B,C,n], w [B,n,3] -> the rounded products fl(g w) [B,C,3n] (slot 3j + k)"""
    b, c, n = g.shape
    return (g.float()[..., None] * w.float()[:, None]).reshape(b, c, 3 * n)


def gather_grad32(g, idx, n, order="ascending"):
    return ordered_scatter(g, idx, n, order)


def group_grad32(g, idx, n, order="ascending"):
    b, c = g.shape[:2]
    return ordered_scatter(g.reshape(b, c, -1), idx.reshape(b, -1), n, order)


def interp_grad32(g, idx, w, m, order="ascending"):
    return ordered_scatter(interp_terms32(g, w), idx.reshape(idx.size(0), -1), m, order)


def pairwise_scatter(terms: torch.Tensor, idx: torch.Tensor, n: int) -> torch.Tensor:
    """mutant: each point's terms summed by a pairwise tree (numpy's np.add.reduce style) instead of one at a time"""
    b, c, j = terms.shape
    t = terms.detach().cpu().numpy().astype(np.float32)
    ix = idx.reshape(b, j).cpu().numpy()
    out = np.zeros((b, c, n), np.float32)

    def tree(v):
        while v.shape[-1] > 1:
            if v.shape[-1] % 2:
                v = np.concatenate([v, np.zeros(v.shape[:-1] + (1,), np.float32)], -1)
            v = (v[..., 0::2] + v[..., 1::2]).astype(np.float32)
        return v[..., 0]

    for f in range(b):
        for i in np.unique(ix[f]):
            if 0 <= i < n:
                out[f, :, i] = tree(t[f][:, ix[f] == i])
    return torch.from_numpy(out).to(terms.device)


def drop_duplicate_slots(idx: torch.Tensor) -> torch.Tensor:
    """mutant input: in each row of a ball index [B,M,S], repeats of an earlier slot point at -1 (dropped)"""
    idx = idx.clone()
    for s in range(1, idx.size(-1)):
        dup = (idx[..., :s] == idx[..., s:s + 1]).any(-1)
        idx[..., s][dup] = -1
    return idx


class Ref64:
    """exact sum, k contributions and S = sum |t| per element (float64); bound = (gamma_{k+2} + gamma_k(U64)) S"""

    def __init__(self, ref, k, s):
        self.ref, self.k, self.s = ref, k, s

    def bound(self):
        k = self.k.expand_as(self.ref)
        return (gamma(k + 2) + gamma(k, U64)) * self.s


def scatter64(terms: torch.Tensor, idx: torch.Tensor, n: int) -> Ref64:
    """terms [B,C,J] (exact products in float64), idx [B,J] -> Ref64 [B,C,n]"""
    b, c, j = terms.shape
    idx = idx.reshape(b, j).long()
    t = terms.double()
    out = torch.zeros((b, c, n), dtype=torch.float64, device=t.device)
    s = torch.zeros_like(out)
    k = torch.zeros((b, 1, n), dtype=torch.float64, device=t.device)
    for f in range(b):
        ok = (idx[f] >= 0) & (idx[f] < n)
        out[f].index_add_(1, idx[f][ok], t[f][:, ok])
        s[f].index_add_(1, idx[f][ok], t[f][:, ok].abs())
        k[f, 0] = torch.bincount(idx[f][ok], minlength=n).double()
    return Ref64(out, k, s)


def interp_terms64(g, w):
    b, c, n = g.shape
    return (g.double()[..., None] * w.double()[:, None]).reshape(b, c, 3 * n)


# ---- adaptive average pooling ---------------------------------------------------------------------------------------
def bin_bounds(o: int, out: int, inn: int, end: str = "ceil"):
    """torch's bin o: [floor(o in / out), ceil((o + 1) in / out)); end="floor" is the mutant"""
    lo = (o * inn) // out
    hi = -((-(o + 1) * inn) // out) if end == "ceil" else ((o + 1) * inn) // out
    return lo, hi


def pool_backward32(g: torch.Tensor, ih: int, iw: int, end: str = "ceil", order: str = "ascending",
                    div: str = "torch") -> torch.Tensor:
    """g [P,OH,OW] f32 -> grad_in [P,ih,iw] f32: the terms of bin (oy, ox) at slots ordered by (oy, ox), then summed by
    ordered_scatter.  A term divides g by the bin's sides in torch's order, width first; div="swapped" is the other
    order."""
    p, oh, ow = g.shape
    g = g.float()
    terms, idx = [], []
    for oy in range(oh):
        y0, y1 = bin_bounds(oy, oh, ih, end)
        for ox in range(ow):
            x0, x1 = bin_bounds(ox, ow, iw, end)
            if y1 <= y0 or x1 <= x0:
                continue
            v = g[:, oy, ox]          # divided by tensors: torch's CUDA division by a Python scalar multiplies by its reciprocal
            kh, kw = torch.full_like(v, float(y1 - y0)), torch.full_like(v, float(x1 - x0))
            t = (v / kw) / kh if div == "torch" else (v / kh) / kw
            pix = (torch.arange(y0, y1)[:, None] * iw + torch.arange(x0, x1)[None]).flatten()
            terms.append(t[:, None].expand(p, pix.numel()))
            idx.append(pix)
    terms = torch.cat(terms, 1)[None]
    idx = torch.cat(idx).to(g.device)[None]
    return ordered_scatter(terms, idx, ih * iw, order)[0].reshape(p, ih, iw)


def _pool_matrix(out: int, inn: int):
    a = np.zeros((out, inn))
    for o in range(out):
        lo, hi = bin_bounds(o, out, inn)
        a[o, lo:hi] = 1.0 / (hi - lo)
    return a


def pool_backward64(g: torch.Tensor, ih: int, iw: int) -> Ref64:
    p, oh, ow = g.shape
    ah = torch.from_numpy(_pool_matrix(oh, ih)).to(g.device)
    aw = torch.from_numpy(_pool_matrix(ow, iw)).to(g.device)
    gd = g.double()
    ref = ah.T @ gd @ aw
    s = ah.T @ gd.abs() @ aw
    k = ((ah > 0).double().sum(0)[:, None] * (aw > 0).double().sum(0)[None])[None]
    return Ref64(ref, k, s)


# ---- bilinear upsampling --------------------------------------------------------------------------------------------
F32 = np.float32


def bilinear_scale(inn: int, out: int, align: bool, scale_factor=None) -> np.float32:
    if align:
        return F32(F32(inn - 1) / F32(out - 1)) if out > 1 else F32(0)
    if scale_factor:
        return F32(1.0 / scale_factor)
    return F32(F32(inn) / F32(out))


def taps(inn: int, out: int, align: bool, scale_factor=None, lam: str = "torch"):
    """[(i1, i1p, l0, l1)] per output index as torch computes them in float32: src = scale o (align_corners) or
    max(fma(scale, o + 0.5, -0.5), 0) -- the fma is torch's CUDA arithmetic, pinned against its forward.
    lam="swapped" is the wrong-align_corners mutant: the other mode's source map."""
    if lam == "swapped":
        align = not align
    scale = bilinear_scale(inn, out, align, scale_factor)
    r = []
    for o in range(out):
        if align:
            src = F32(scale * F32(o))
        else:
            src = F32(np.float64(scale) * np.float64(F32(F32(o) + F32(0.5))) - 0.5)   # fma: one rounding
            src = max(src, F32(0))
        i1 = int(src)
        p = 1 if i1 < inn - 1 else 0
        l1 = F32(src - F32(i1))
        r.append((i1, p, F32(F32(1) - l1), l1))
    return r


def upsample_backward32(g: torch.Tensor, ih: int, iw: int, align: bool, scale_factor=None, lam="torch",
                        order: str = "ascending") -> torch.Tensor:
    """g [P,OH,OW] f32 -> grad_in [P,ih,iw] f32: the four tap terms of output o at slots 4o .. 4o + 3 in torch's tap
    order, summed by ordered_scatter"""
    p, oh, ow = g.shape
    th = np.array([t for t in taps(ih, oh, align, scale_factor, lam)], dtype=object)
    tw = np.array([t for t in taps(iw, ow, align, scale_factor, lam)], dtype=object)
    h1 = np.array([t[0] for t in th], np.int64); hp = np.array([t[1] for t in th], np.int64)
    lh = np.stack([np.array([t[2] for t in th], F32), np.array([t[3] for t in th], F32)])       # [2, OH]
    w1 = np.array([t[0] for t in tw], np.int64); wp = np.array([t[1] for t in tw], np.int64)
    lw = np.stack([np.array([t[2] for t in tw], F32), np.array([t[3] for t in tw], F32)])       # [2, OW]
    ys = np.stack([h1, h1 + hp])                                                                # [2, OH]
    xs = np.stack([w1, w1 + wp])                                                                # [2, OW]
    idx = np.empty((oh, ow, 4), np.int64)
    lam2 = np.empty((oh, ow, 4), F32)
    for t, (a, c) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        idx[..., t] = ys[a][:, None] * iw + xs[c][None]
        lam2[..., t] = (lh[a][:, None] * lw[c][None]).astype(F32)                              # fl(lh lw)
    lam2 = torch.from_numpy(lam2.reshape(-1)).to(g.device)
    terms = (g.float().reshape(p, oh * ow, 1) * lam2.reshape(1, oh * ow, 4)).reshape(1, p, oh * ow * 4)
    idx = torch.from_numpy(idx.reshape(1, -1)).to(g.device)
    return ordered_scatter(terms, idx, ih * iw, order)[0].reshape(p, ih, iw)


def _interp_matrix(inn: int, out: int, align: bool, scale_factor=None, lam="torch"):
    a = np.zeros((out, inn))
    cnt = np.zeros((out, inn))
    for o, (i1, p, l0, l1) in enumerate(taps(inn, out, align, scale_factor, lam)):
        a[o, i1] += float(l0)
        a[o, i1 + p] += float(l1)
        cnt[o, i1] += 1
        cnt[o, i1 + p] += 1
    return a, cnt


def upsample_backward64(g: torch.Tensor, ih: int, iw: int, align: bool, scale_factor=None, lam="torch") -> Ref64:
    p, oh, ow = g.shape
    ah, ch = (torch.from_numpy(x).to(g.device) for x in _interp_matrix(ih, oh, align, scale_factor, lam))
    aw, cw = (torch.from_numpy(x).to(g.device) for x in _interp_matrix(iw, ow, align, scale_factor, lam))
    gd = g.double()
    return Ref64(ah.T @ gd @ aw, (ch.sum(0)[:, None] * cw.sum(0)[None])[None], ah.T @ gd.abs() @ aw)


def upsample_forward_onehot(ih: int, iw: int, oh: int, ow: int, align: bool, scale_factor=None):
    """the forward of every one-hot input where no two taps of an output coincide: {(y, x): [OH,OW] f32} with
    out[oy,ox] = fl(lh lw) for the tap on (y, x), NaN where taps coincide (torch's forward sums them there in an
    unpinned order).  Pins the source indices and lambdas against torch's forward."""
    th, tw = taps(ih, oh, align, scale_factor), taps(iw, ow, align, scale_factor)
    res = {}
    for y in range(ih):
        for x in range(iw):
            out = np.zeros((oh, ow), np.float32)
            for oy, (h1, hp, h0l, h1l) in enumerate(th):
                for ox, (w1, wp, w0l, w1l) in enumerate(tw):
                    if hp == 0 or wp == 0:
                        if y in (h1, h1 + hp) and x in (w1, w1 + wp):
                            out[oy, ox] = np.nan
                        continue
                    for yy, lh in ((h1, h0l), (h1 + 1, h1l)):
                        for xx, lw in ((w1, w0l), (w1 + 1, w1l)):
                            if yy == y and xx == x:
                                out[oy, ox] = F32(lh * lw)
            res[(y, x)] = out
    return res


# ---- checks ---------------------------------------------------------------------------------------------------------
def check_bound(got: torch.Tensor, r: Ref64, what: str = "") -> float:
    """|got - ref| <= bound everywhere (NaN outside); k = 0 must be +0.0.  Returns the worst |got - ref| / bound."""
    err = (got.double() - r.ref).abs()
    bound = r.bound()
    bad = ~(err <= bound)
    k = r.k.expand_as(r.ref)
    bad |= (k == 0) & (got.float().contiguous().view(torch.int32) != 0)
    pos = bound > 0
    worst = float((err[pos] / bound[pos]).max()) if bool(pos.any()) else 0.0
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        ix = tuple(int(v) for v in np.unravel_index(i, tuple(bad.shape)))
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the bound, first at {ix}: "
                             f"got {float(got[ix])!r} ref {float(r.ref[ix])!r} bound {float(bound[ix]):.3g}")
    return worst


def check_bits(got: torch.Tensor, want: torch.Tensor, what: str = "") -> None:
    """bit equality (the fixed-order contract)"""
    gb = got.float().contiguous().view(torch.int32)
    wb = want.float().contiguous().view(torch.int32)
    if gb.shape != wb.shape or not torch.equal(gb, wb):
        n = int((gb != wb).sum()) if gb.shape == wb.shape else -1
        raise AssertionError(f"{what}: {n} elements differ in bits from the restatement")


def cancelling_terms(c: int, j: int, seed: int = 0) -> torch.Tensor:
    """terms [1,c,j] whose sum depends on the order: big values that cancel plus small ones"""
    gen = torch.Generator().manual_seed(seed)
    t = torch.randn((1, c, j), generator=gen)
    t[..., ::3] *= 2.0 ** 20
    return t
