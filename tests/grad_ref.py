"""Float64 references of the three PointNet++ gradient ops with an element-wise bound, and wrong references
("mutants") they must reject (test infrastructure, no conftest).  Everything is torch, float64, on whatever device the
operands live on.

The ops are atomic scatter-adds (csrc/pn2_ops.cu):
  * gather_points_grad:      out[b,c,idx[b,j]]   += g[b,c,j]
  * group_points_grad:       the same over the M*S slots of idx[b,M,S]
  * three_interpolate_grad:  out[b,c,idx[b,j,t]] += fl32(g[b,c,j] * w[b,j,t])
Each reference returns, per output element, the exact sum (float64: the product of two float32 values is exact in
float64), k = the number of contributions and S = the sum of their absolute values.  Any order of k fp32 additions
onto the zero the memset wrote is within gamma_k * S of the exact sum, gamma_k = k u / (1 - k u), u = 2^-24 (Higham,
Accuracy and Stability of Numerical Algorithms, 2nd ed., eq. 4.4).  For the interpolation the one rounding of each
product g*w moves each term by <= u |t|, which the same gamma_k covers: u S + gamma_{k-1} (1 + u) S <= gamma_k S.  The
float64 sum itself is within gamma_k(2^-53) S of the exact one; that is added to the bound.

Inside the bound two cases are exact: k = 0 is the memset's +0.0, and k = 1 is 0 + t, the reference's own value
rounded to float32 (for interpolate: fl32(g*w), the torch float32 product; a -0.0 product becomes +0.0 on the zero).
With integer-valued g (and dyadic weights) every partial sum is an integer (a multiple of the weights' denominator) far
below 2^24, so any order gives the exact sum: `check(..., exact=True)` demands bit equality everywhere.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

U32 = 2.0 ** -24
U64 = 2.0 ** -53


def gamma(k: torch.Tensor, u: float = U32) -> torch.Tensor:
    ku = k.double() * u
    return ku / (1.0 - ku)


@dataclass
class Ref:
    """exact sum [B,C,N] f64, k [B,1,N] int64 (the same for every channel), s = sum |t| [B,C,N] f64"""
    ref: torch.Tensor
    k: torch.Tensor
    s: torch.Tensor

    def bound(self) -> torch.Tensor:
        return (gamma(self.k) + gamma(self.k, U64)) * self.s


def _scatter(terms: torch.Tensor, idx: torch.Tensor, n: int) -> Ref:
    """terms [B,C,J] f64, idx [B,J] -> Ref: out[b,c,idx[b,j]] += terms[b,c,j]"""
    b, c, _ = terms.shape
    idx = idx.long()
    out = torch.zeros((b, c, n), dtype=torch.float64, device=terms.device)
    s = torch.zeros_like(out)
    k = torch.zeros((b, 1, n), dtype=torch.int64, device=terms.device)
    for f in range(b):
        out[f].index_add_(1, idx[f], terms[f])
        s[f].index_add_(1, idx[f], terms[f].abs())
        k[f, 0] = torch.bincount(idx[f], minlength=n)
    return Ref(out, k, s)


def gather_grad(g: torch.Tensor, idx: torch.Tensor, n: int) -> Ref:
    """g [B,C,M], idx [B,M] -> Ref [B,C,n]"""
    return _scatter(g.double(), idx, n)


def group_grad(g: torch.Tensor, idx: torch.Tensor, n: int) -> Ref:
    """g [B,C,M,S], idx [B,M,S] -> Ref [B,C,n]"""
    b, c = g.shape[:2]
    return _scatter(g.double().reshape(b, c, -1), idx.reshape(b, -1), n)


def interp_terms(g: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """g [B,C,n], w [B,n,3] -> the exact products [B,C,n*3] (slot-major per point, as idx.reshape(B, -1))"""
    b, c, n = g.shape
    return (g.double()[..., None] * w.double()[:, None]).reshape(b, c, n * 3)


def interp_grad(g: torch.Tensor, idx: torch.Tensor, w: torch.Tensor, m: int) -> Ref:
    """g [B,C,n], idx [B,n,3], w [B,n,3] -> Ref [B,C,m]"""
    return _scatter(interp_terms(g, w), idx.reshape(idx.size(0), -1), m)


def _bits(x: torch.Tensor) -> torch.Tensor:
    return x.float().contiguous().view(torch.int32)


def check(got: torch.Tensor, r: Ref, what: str = "", exact: bool = False) -> float:
    """assert |got - ref| <= gamma_k S everywhere, k = 0 bit-equal to +0.0 and k = 1 bit-equal to fl32(ref); with
    exact=True (integer-valued inputs) got must equal the reference bit for bit everywhere.  Returns and prints the
    worst |got - ref| / bound over the elements with a non-zero bound."""
    assert got.dtype == torch.float32 and got.shape == r.ref.shape, (what, got.dtype, tuple(got.shape))
    k = r.k.expand_as(r.ref)
    err = (got.double() - r.ref).abs()
    bound = torch.zeros_like(err) if exact else r.bound()
    bad = ~(err <= bound)                                          # NaN in got counts as outside
    gb, rb = _bits(got), _bits(r.ref)
    bad |= (k == 0) & (gb != 0)
    bad |= (k == 1) & (gb != rb)
    if exact:
        bad |= gb != rb
    pos = bound > 0
    worst = float((err[pos] / bound[pos]).max()) if bool(pos.any()) else 0.0
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        ix = tuple(int(x) for x in np.unravel_index(i, tuple(bad.shape)))
        raise AssertionError(
            f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the bound, first at {ix}: got "
            f"{float(got[ix])!r} ref {float(r.ref[ix])!r} k {int(k[ix])} sum|t| {float(r.s[ix]):.6g} bound "
            f"{float(bound[ix]):.3g}; worst |got - ref| / bound {worst:.3g}")
    print(f"{what}: worst |got - ref| / bound {worst:.3g} (max k {int(r.k.max()) if r.k.numel() else 0})")
    return worst


def check_pair(a: torch.Tensor, b: torch.Tensor, r: Ref, what: str = "") -> None:
    """two results of the same op on the same inputs (different atomic orders) agree within twice the bound"""
    err = (a.double() - b.double()).abs()
    bad = ~(err <= 2 * r.bound())
    if bool(bad.any()):
        ix = tuple(int(x) for x in np.unravel_index(int(bad.flatten().nonzero()[0]), tuple(bad.shape)))
        raise AssertionError(f"{what}: {int(bad.sum())} elements outside the bound, first at {ix}: "
                             f"{float(a[ix])!r} vs {float(b[ix])!r}")


def channel_slices(c: int, other_ctas: int, sm_count: int) -> int:
    """grid.y of the three grad launches (pn2_ops.cu channel_slices): channel l runs in slice l % grid.y"""
    want = -(-4 * sm_count // max(other_ctas, 1))
    return max(1, min(want, c, 65535))


# ---- mutants: float32 results of plausible kernel mistakes on the same inputs ----------------------------------------
def mut_group_dedup(g: torch.Tensor, idx: torch.Tensor, n: int) -> torch.Tensor:
    """group_points_grad counting a point once per centre: the padded duplicate slots of a ball row dropped"""
    idx = idx.long()
    keep = torch.ones(idx.shape, dtype=torch.bool, device=idx.device)
    for s in range(1, idx.size(-1)):
        keep[..., s] = ~(idx[..., :s] == idx[..., s:s + 1]).any(-1)
    return group_grad(g * keep[:, None].to(g.dtype), idx, n).ref.float()


def mut_frames(r: Ref, mode: str) -> torch.Tensor:
    """'frame0': every frame scattered with frame 0's offset (all frames land in frame 0); 'shift': frame b's
    contributions land in frame b + 1 (the last wraps to 0)"""
    if mode == "frame0":
        out = torch.zeros_like(r.ref)
        out[0] = r.ref.sum(0)
        return out.float()
    assert mode == "shift"
    return torch.roll(r.ref, 1, 0).float()


def mut_drop_channels(r: Ref, channels) -> torch.Tensor:
    """the given channels left at the memset's zero (the last channel, or one channel slice: range(y, C, grid.y))"""
    out = r.ref.clone()
    out[:, list(channels)] = 0
    return out.float()


def mut_swap_nn_weights(w: torch.Tensor) -> torch.Tensor:
    """weights of NN slots 1 and 2 exchanged (feed to interp_grad)"""
    return w[..., [0, 2, 1]].contiguous()


def mut_drop_one(terms: torch.Tensor, idx: torch.Tensor, r: Ref) -> torch.Tensor:
    """one contribution (the largest |t| of each channel) removed from the element with the largest k.
    terms [B,C,J] as passed to the scatter (g, g reshaped, or interp_terms), idx [B,J]"""
    idx = idx.long()
    kk = r.k[:, 0]
    f, a = (int(x) for x in np.unravel_index(int(kk.flatten().argmax()), tuple(kk.shape)))
    sel = (idx[f] == a).nonzero().flatten()
    t = terms[f][:, sel].double()                                  # [C, k]
    pick = t.abs().argmax(1)
    out = r.ref.clone()
    out[f, :, a] -= t.gather(1, pick[:, None])[:, 0]
    return out.float()


def mut_reference_wrapper(g, idx, w, m: int) -> np.ndarray:
    """what the reference's three_interpolate_grad returns (interpolate.cpp:89-93): the FORWARD kernel launched as
    (b, c, m := grad_out.size(2), n := m) on grad_out, so out[b,l,j] = sum_t g[b,l,i_t] w_t with the idx / weight rows
    read at the forward's frame stride m*3 (restated in numpy)"""
    g = np.asarray(g, np.float64)
    b, c, n = g.shape
    fi = np.asarray(idx).reshape(-1)[:b * m * 3].reshape(b, m, 3).astype(np.int64)
    fw = np.asarray(w, np.float64).reshape(-1)[:b * m * 3].reshape(b, m, 3)
    out = np.zeros((b, c, m))
    for f in range(b):
        out[f] = (g[f][:, fi[f]] * fw[f][None]).sum(-1)
    return out.astype(np.float32)
