"""The pieces of the float64 twin of a PVN3D training step (tests/test_train_step_f64_gpu.py) -- test infrastructure,
importable without a GPU.

  * replay ops: pure-torch stand-ins for the module-level ops of the reference's lib.pointnet2_utils.pointnet2_utils.
    `recorder` wraps the discrete ops (FPS, ball query, 3-NN) so that a package step records its choices; `twin`
    returns ops that replay those choices and compute gather / group / interpolate and their gradients in torch.  The
    arithmetic follows the 16-bit contract of the package's kernels (include/pvn3d_b200.h): float32 or float64 inputs
    are computed in their own precision; float16 / bfloat16 inputs are widened to float32, computed there, and each
    output element (forward value or gradient) is rounded once to the input's dtype.  A plain torch gather on a 16-bit
    tensor would instead add its scatter gradient in 16 bits, rounding after every term.
  * the error statistic of a parameter gradient against float64 and the bound an arm must meet relative to its twin.
  * the wrong gradients ("mutants") the step's check must reject, as functions of the op's inputs.
"""
from __future__ import annotations

import math

import torch

DISCRETE = ("furthest_point_sample", "ball_query", "three_nn")
U16 = (torch.float16, torch.bfloat16)


def acc_dtype(dt: torch.dtype) -> torch.dtype:
    """the precision an op on `dt` computes in: float32 for the 16-bit dtypes, the dtype itself otherwise"""
    return torch.float32 if dt in U16 else dt


def _gather_cols(features: torch.Tensor, flat_idx: torch.Tensor) -> torch.Tensor:
    """features [B,C,N], flat_idx [B,J] -> [B,C,J]"""
    b, c = features.shape[:2]
    return features.gather(2, flat_idx.long()[:, None].expand(b, c, flat_idx.size(1)))


def _scatter_cols(g: torch.Tensor, flat_idx: torch.Tensor, n: int) -> torch.Tensor:
    """the adjoint of _gather_cols: g [B,C,J] summed into [B,C,n] in g's dtype"""
    b, c = g.shape[:2]
    out = torch.zeros((b, c, n), dtype=g.dtype, device=g.device)
    return out.scatter_add_(2, flat_idx.long()[:, None].expand(b, c, flat_idx.size(1)), g)


class Group(torch.autograd.Function):
    """grouping_operation / gather_operation: features [B,C,N], idx [B,*] -> [B,C,*] (an exact copy); the gradient is
    summed in acc_dtype and rounded once"""

    @staticmethod
    def forward(ctx, features, idx):
        b, c, n = features.shape
        ctx.save_for_backward(idx)
        ctx.n = n
        return _gather_cols(features, idx.reshape(b, -1)).reshape(b, c, *idx.shape[1:])

    @staticmethod
    def backward(ctx, g):
        (idx,) = ctx.saved_tensors
        b, c = g.shape[:2]
        acc = _scatter_cols(g.to(acc_dtype(g.dtype)).reshape(b, c, -1), idx.reshape(b, -1), ctx.n)
        return acc.to(g.dtype), None


class Interp(torch.autograd.Function):
    """three_interpolate: features [B,C,M], idx / weight [B,n,3] -> [B,C,n] = sum_t w_t f[idx_t] computed in acc_dtype
    and rounded once; the gradient scatters g w_t in acc_dtype and rounds once"""

    @staticmethod
    def forward(ctx, features, idx, weight):
        b, c, m = features.shape
        n = idx.size(1)
        acc = acc_dtype(features.dtype)
        w = weight.to(acc)
        ctx.save_for_backward(idx, w)
        ctx.m = m
        f = _gather_cols(features.to(acc), idx.reshape(b, -1)).reshape(b, c, n, 3)
        return (f * w[:, None]).sum(-1).to(features.dtype)

    @staticmethod
    def backward(ctx, g):
        idx, w = ctx.saved_tensors
        b, c, n = g.shape
        terms = (g.to(w.dtype)[..., None] * w[:, None]).reshape(b, c, n * 3)
        return _scatter_cols(terms, idx.reshape(b, -1), ctx.m).to(g.dtype), None, None


def recorder(log: dict, ops: dict) -> dict:
    """the discrete ops `ops` (name -> callable), each appending its output to log[name]"""
    def wrap(name):
        def fn(*a):
            out = ops[name](*a)
            log[name].append(out)
            return out
        return fn
    return {k: wrap(k) for k in DISCRETE}


def twin(log: dict, f64: bool) -> dict:
    """pure-torch ops replaying the recorded FPS / ball-query / 3-NN choices.  f64: the 3-NN distances are recomputed
    from the float64 coordinates (the reference's three_nn returns distances, not their squares).  Otherwise the
    recorded float32 distances are replayed too, so an error in them would be shared by a twin and the package arm it
    bounds: the distances are held to the oracle by the three_nn tests, and the fp32 twin's own error against float64
    is bounded in absolute terms by tests/test_train_step_f64_gpu.py."""
    its = {k: iter(v) for k, v in log.items()}

    def nn(unknown, known):
        dist, idx = next(its["three_nn"])
        if f64:
            b, n = idx.shape[:2]
            k = known.detach().gather(1, idx.long().reshape(b, -1, 1).expand(b, n * 3, 3)).reshape(b, n, 3, 3)
            dist = (unknown.detach()[:, :, None] - k).square().sum(-1).sqrt()
        return dist, idx

    return {"furthest_point_sample": lambda xyz, npoint: next(its["furthest_point_sample"]),
            "ball_query": lambda radius, nsample, xyz, new_xyz: next(its["ball_query"]),
            "three_nn": nn, "gather_operation": Group.apply, "grouping_operation": Group.apply,
            "three_interpolate": Interp.apply}


# ---- the statistic and the bound -------------------------------------------------------------------------------------
def err(g: torch.Tensor, g64: torch.Tensor, scale=None) -> tuple[float, float]:
    """(mean, 99.9th percentile) of |g - g64| / scale; scale = mean |g64| unless given (a number, or a tensor that
    broadcasts against g: sum |term| of each element of a gradient whose sum cancels)"""
    s = float(g64.abs().mean()) if scale is None else scale
    e = ((g.double() - g64).abs() / s).flatten()
    return float(e.mean()), float(e.kthvalue(max(1, math.ceil(0.999 * e.numel()))).values)


def within(ea, eb, floor: float) -> bool:
    """an arm's (mean, p99.9) error within 2 x its twin's + floor, both statistics"""
    return all(a <= 2 * b + floor for a, b in zip(ea, eb))


def ratio(ea, eb, floor: float) -> float:
    """how much of the bound an arm uses: max over the two statistics of (error - floor) / (2 x twin error)"""
    return max((a - floor) / max(2 * b, 1e-300) for a, b in zip(ea, eb))


FAMILIES = (("cnn.", "CNN"), ("pointnet2.", "PointNet++"), ("rgbd_feat.", "DenseFusion"), ("", "heads"))


def family(name: str) -> str:
    return next(f for p, f in FAMILIES if name.startswith(p))


# ---- mutants ---------------------------------------------------------------------------------------------------------
def first_of_run(idx: torch.Tensor) -> torch.Tensor:
    """bool [B,J] over the flattened slots of idx [B,*]: True at the lowest slot of each point's run (the first term of
    every output element the ordered grad sums).  Sort and gather only, so it runs under
    torch.use_deterministic_algorithms(True)."""
    flat = idx.reshape(idx.size(0), -1).long()
    key, order = torch.sort(flat, dim=1, stable=True)
    head = torch.ones_like(key, dtype=torch.bool)
    head[:, 1:] = key[:, 1:] != key[:, :-1]
    return head.gather(1, torch.argsort(order, dim=1))


def drop_first_of_run(g: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """the group grad's input with the first slot of every run zeroed: g [B,C,M,S], idx [B,M,S]"""
    keep = ~first_of_run(idx).reshape(idx.shape)
    return g * keep[:, None].to(g.dtype)


def swap_pairs(weight: torch.Tensor) -> torch.Tensor:
    """the interpolation weights of points j and j+1 exchanged (j even; an odd last point keeps its own): [B,n,3]"""
    n = weight.size(1)
    perm = torch.arange(n, device=weight.device)
    top = n - n % 2
    perm[:top] = perm[:top].view(-1, 2).flip(1).reshape(-1)
    return weight[:, perm].contiguous()


LOSS_SCALE_MUTANT = 1.0 + 2.0 ** -8
