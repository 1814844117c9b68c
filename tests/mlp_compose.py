"""What the fused shared-MLP kernels compute, composed from torch and the dense layer (test infrastructure, no conftest).

Each fused kernel builds the rows of its first contracted layer on chip, TF32-rounds them as the dense layer's producer
does, and runs its layers with the dense layer's MMA order and epilogue.  The compositions below build the same fp32 rows
in torch with the same arithmetic and feed them to `mlp.mlp_dense`, so each fused result must equal its composition bit
for bit:

  * SA (sa_fact2, sa_fact2w): rows relu(U[idx] - V), one fp32 subtraction and a max; layer 2 rounded to TF32, layer 3,
    then the max over the nsample rows of each centre.  The kernels take that max over the raw accumulators and add the
    bias afterwards; x -> tf32(relu(fl(x + b))) is monotone non-decreasing, so taking it after the epilogue gives the same
    bits.
  * FP2-FP4 (fp2): rows [three_interpolate(known) | skip[:, :c1] | 0], where pvn3d_three_interpolate evaluates the
    kernels' fma(p3,w3, fma(p1,w1, p2*w2)); layer 1 rounded to TF32, layer 2.
  * FP1 (fp_fact2): S = W1s . table + b1 (the dense layer without ReLU), rows relu(three_interpolate(P) + S) with one
    plain add, layer 2, transposed to [b, 128, n] per frame.
The transposes around three_interpolate move values and change none.
"""
from __future__ import annotations

import torch

from pvn3d_b200 import _ext, mlp


def _interpolate(known_pm: torch.Tensor, nn_idx: torch.Tensor, nn_w: torch.Tensor) -> torch.Tensor:
    """known_pm [b, m, c] point-major, nn_idx / nn_w [b, n, 3] -> [b * n, c] point-major (pvn3d_three_interpolate)"""
    b, n = nn_idx.shape[0], nn_idx.shape[1]
    cn = _ext.three_interpolate(known_pm.transpose(1, 2).contiguous(), nn_idx.contiguous(), nn_w.contiguous())
    return cn.transpose(1, 2).reshape(b * n, -1).contiguous()   # b = 1: reshape is a transposed view


def sa_fact2(u, v, idx, n, l2, l3, round_out=False, out=None, col0=0):
    """mlp_sa_fact2 / mlp_sa_fact2w: u [b*n, ldu], v [b*m, ldu], idx [b, m, ns] -> [b*m, l3.n_pad] (or written into the
    columns col0 .. col0 + l3.n_pad of out)"""
    b, m, ns = idx.shape
    bi = torch.arange(b, device=u.device)[:, None, None]
    rows = (u.view(b, n, -1)[bi, idx.long()] - v.view(b, m, 1, -1)).clamp_min(0).reshape(-1, u.size(-1))
    h = mlp.mlp_dense(rows, l2, round_out=True)
    y = mlp.mlp_dense(h, l3, a_tf32=True, round_out=round_out)
    want = y.view(b * m, ns, -1).amax(1)
    if out is None:
        return want
    out[:, col0:col0 + want.size(-1)] = want
    return out


def fp2(known, skip, nn_idx, nn_w, lds, c1, l1, l2, round_out=False, reserve=0):
    """mlp_fp2: known [b, m, c2], skip rows lds apart (c1 valid columns), nn_idx / nn_w [b, n, 3] -> [b*n, l2.n_pad]"""
    interp = _interpolate(known, nn_idx, nn_w)
    rows_n, c2 = interp.shape
    width = (c2 + c1 + 3) // 4 * 4                          # the dense layer reads whole groups of four columns
    rows = torch.zeros((rows_n, width), dtype=torch.float32, device=known.device)
    rows[:, :c2] = interp
    if c1:
        rows[:, c2:c2 + c1] = torch.as_strided(skip, (rows_n, c1), (lds, 1))
    h = mlp.mlp_dense(rows, l1, round_out=True, reserve=reserve)
    return mlp.mlp_dense(h, l2, a_tf32=True, round_out=round_out, reserve=reserve)


def fp_fact2(p, table, nn_idx, nn_w, m, ls, l2, reserve=0):
    """mlp_fp_fact2: p [b*m, 128], the SA1 factor table [b*n, ls.k_pad], nn_idx / nn_w [b, n, 3] -> [b, 128, n]"""
    b, n = nn_idx.shape[0], nn_idx.shape[1]
    s = mlp.mlp_dense(table, ls, relu=False, a_tf32=True, reserve=reserve)
    rows = (_interpolate(p.view(b, m, -1), nn_idx, nn_w) + s).clamp_min(0)
    pm = mlp.mlp_dense(rows, l2, reserve=reserve)
    return pm.view(b, n, -1).transpose(1, 2).contiguous()
