"""Float64 reference of the batched mean-shift (test infrastructure).

What `csrc/meanshift.cu` computes, restated independently of the kernels:

* the exact part -- inlier counts, the first-index arg-max `max_idx`, `labels` -- with the oracle's own fp32 CPU
  `torch.norm` ops (`oracle.meanshift_oracle.density_labels`, the contraction `fma(z,z,fma(y,y,x*x))` the reference's
  CPU run uses), so it must agree with the kernels bit for bit;
* the iterations in float64: every point is a seed, C <- sum_j w_ij A_j / sum_j w_ij with w_ij = exp(-|C_i-A_j|^2 /
  (2 bw^2)), and the reference's stop rule: T is the first iteration whose largest shift is below float32(bw * 1e-3),
  or the iteration after max_iter.  Returned per fit: T, the largest shift at every iteration and the trajectory of
  the star (the seed at max_idx) up to T + 1.

The all-seed sweep costs n^2 per iteration, so it runs on the GPU (float64 bmm + exp), fits of similar size batched
and chunked so that one [F, m, m] float64 matrix stays below `MAX_ELEMS` elements.

The centre bound.  The kernels sweep in fp32 about the star's input point: w = ex2.approx(k|a'|^2 + k|c'|^2 -
2k a'.c') with k = -log2(e) / (2 bw^2).  For the pairs that carry the star's weight (|a'|, |c'| within a few bw)
the argument is a sum of terms of magnitude <= ~40 rounded a few times (<= 2^-17 absolute) and ex2.approx adds
<= 2^-22 relative, so a weight is off by <= ~2^-16 relative and one sweep moves the weighted mean by <= 2^-16 of the
spread of its support (~2 bw).  Near its mode a sweep contracts earlier errors, so the star's error stays within a
small multiple of that: 2^-15 bw.  The fp32 centre itself and the final `+ origin` add 2^-20 |C|.
    bound(C, bw) = 2^-20 |C| + 2^-15 bw
At the tested clouds (|C| ~ 0.9 m, bw <= 0.16) this is below 1e-5 |C|: ten times tighter than the 1e-4 relative
parity bar; `test_meanshift_f64_gpu` asserts it case by case.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle.meanshift_oracle import density_labels

MAX_ELEMS = 1 << 27          # elements of one batched [F, m, m] float64 matrix (1 GiB)
DELTA_REL = 1e-5             # certified mode: the returned centre is within delta = 1e-5 bw of C_T (DESIGN section 5)


def centre_bound(c, bw: float) -> float:
    """the stated bound on |ctr_kernel - C_64| at the same iteration count (module docstring)"""
    return 2.0 ** -20 * float(np.linalg.norm(np.asarray(c, np.float64))) + 2.0 ** -15 * float(bw)


def shift_tol(A: np.ndarray, max_idx: int, bw: float) -> float:
    """bound on the kernels' error in a seed's shift.  The sweep's exponent k|a'|^2 + k|c'|^2 - 2k a'.c' is summed
    in fp32 from terms up to 2|k|R^2 (R = the largest distance of a point from the star's input point, about which
    the kernels centre), so it is off by <= 2^-20 |k| R^2; with ex2.approx that makes a weight off by
    <= ln2 2^-20 |k| R^2 + 2^-22 relative.  Pairs carrying weight lie within ~4 bw, so a shift moves by at most
    8 bw times that.  For a creeping outlier seed the shift is a small difference of large weighted sums: this,
    not the 1e-4 relative of the reference rule's own rounding, is how close to the threshold the kernels' T can
    legitimately step off the float64 T."""
    A = np.asarray(A, np.float64)
    if len(A) == 0:
        return 0.0
    R2 = float(((A - A[max_idx]) ** 2).sum(1).max())
    k = 1.4426950408889634 / (2.0 * float(bw) ** 2)
    return 8.0 * float(bw) * (np.log(2.0) * 2.0 ** -20 * k * R2 + 2.0 ** -22)


def stop_thresh(bw: float) -> float:
    """the stop threshold as the kernels hold it: float32(bw * 1e-3)"""
    return float(np.float32(bw * 1e-3))


def exact_part(A: np.ndarray, bw: float):
    """A [n,3] float32 -> (num_in [n] int64, max_idx int, labels [n] bool); n == 0 -> empty, -1"""
    A = np.ascontiguousarray(A, np.float32)
    if len(A) == 0:
        return np.zeros(0, np.int64), -1, np.zeros(0, bool)
    num_in, max_idx, labels = density_labels(torch.from_numpy(A), bw)
    return num_in.numpy(), int(max_idx), labels.numpy()


def _groups(sizes, max_elems):
    """indices of the non-empty fits, sorted by size, cut into batches of similar size within max_elems"""
    order = [i for i in np.argsort(sizes, kind="stable") if sizes[i] > 0]
    out, cur = [], []
    for i in order:
        m = sizes[i]
        if cur and ((len(cur) + 1) * m * m > max_elems or m > 1.25 * sizes[cur[0]] + 64):
            out.append(cur)
            cur = []
        cur.append(i)
    if cur:
        out.append(cur)
    return out


def iterate_f64(clouds, bw: float, max_iter: int, max_idx, device, max_elems: int = MAX_ELEMS):
    """clouds: list of [n_i,3] float32 arrays; max_idx: the star of each (from exact_part).
    Returns a list of dicts (None for empty clouds): T, shifts [T+2] (shifts[it] = largest shift of iteration it,
    shifts[0] = nan), traj [T+2, 3] float64 world coordinates (traj[0] = the star's input point)."""
    sizes = [len(c) for c in clouds]
    res = [None] * len(clouds)
    thr = stop_thresh(bw)
    inv = -0.5 / (float(bw) * float(bw))
    for grp in _groups(sizes, max_elems):
        F, m = len(grp), max(sizes[i] for i in grp)
        A = torch.zeros((F, m, 3), dtype=torch.float64)
        valid = torch.zeros((F, m), dtype=torch.bool)
        org = torch.zeros((F, 3), dtype=torch.float64)
        star = torch.tensor([max_idx[i] for i in grp], dtype=torch.int64)
        for g, i in enumerate(grp):
            a = torch.from_numpy(np.asarray(clouds[i], np.float32).astype(np.float64))
            org[g] = a[max_idx[i]]
            A[g, :sizes[i]] = a - org[g]
            valid[g, :sizes[i]] = True
        A, valid, org, star = A.to(device), valid.to(device), org.to(device), star.to(device)
        ar = torch.arange(F, device=device)
        a2 = (A * A).sum(-1)
        wmask = valid.to(torch.float64)[:, None, :]
        C = A.clone()
        T = torch.full((F,), -1, dtype=torch.int64, device=device)
        traj, shifts = [C[ar, star].clone()], [torch.full((F,), float("nan"), dtype=torch.float64, device=device)]
        it = 0
        while True:
            it += 1
            c2 = (C * C).sum(-1)
            d2 = (c2[:, :, None] + a2[:, None, :] - 2.0 * torch.bmm(C, A.transpose(1, 2))).clamp_(min=0.0)
            w = torch.exp(d2.mul_(inv)).mul_(wmask)
            del d2
            newC = torch.bmm(w, A) / w.sum(-1, keepdim=True)
            del w
            sh = torch.linalg.vector_norm(newC - C, dim=-1).masked_fill_(~valid, 0.0).amax(-1)
            C = newC
            traj.append(C[ar, star].clone())
            shifts.append(sh)
            stop = (T < 0) & ((sh < thr) | (it > max_iter))
            T = torch.where(stop, torch.full_like(T, it), T)
            if bool((T >= 0).all()) and it >= int(T.max()) + 1:
                break
        traj = (torch.stack(traj, 1) + org[:, None, :]).cpu().numpy()
        shifts = torch.stack(shifts, 1).cpu().numpy()
        T = T.cpu().numpy()
        for g, i in enumerate(grp):
            t = int(T[g])
            res[i] = dict(T=t, shifts=shifts[g, :t + 2], traj=traj[g, :t + 2])
    return res


def reference(clouds, bw: float, max_iter: int, device):
    """exact part + float64 iterations of every cloud: list of dicts (num_in, max_idx, labels, and for non-empty
    clouds T, shifts, traj)"""
    out = []
    for A in clouds:
        num_in, mi, labels = exact_part(A, bw)
        out.append(dict(num_in=num_in, max_idx=mi, labels=labels, shift_tol=shift_tol(A, mi, bw)))
    its = iterate_f64(clouds, bw, max_iter, [o["max_idx"] for o in out], device)
    for o, r in zip(out, its):
        if r is not None:
            o.update(r)
    return out


def t_near_threshold(ref, t: int, bw: float, rel: float = 1e-4) -> bool:
    """whether the float64 largest shift of iteration t - 1 or t lies within rel of the stop threshold, or within
    the kernels' shift error bound (shift_tol) of it"""
    thr = stop_thresh(bw)
    tol = max(rel * thr, ref.get("shift_tol", 0.0))
    for k in (t - 1, t):
        if 1 <= k < len(ref["shifts"]) and abs(ref["shifts"][k] - thr) <= tol:
            return True
    return False


def check_fit(mode: str, ref, ctr, iters: int, bw: float, rel: float = 1e-4):
    """The float64 checks of one fit; returns (ok, ratio, message).  ratio = |ctr - C_ref| / allowed.
    strict / no_freeze: |T - T64| <= 1, T == T64 unless the float64 shift at T-1 or T is within rel (or the
                        kernels' shift error bound) of the threshold, and the centre within the bound of the
                        float64 star at the kernel's own T
    early_exit / certified: iters <= T64 + 1 and the centre within delta + bound of the star at T64"""
    T64 = ref["T"]
    ctr = np.asarray(ctr, np.float64)
    if mode in ("strict", "no_freeze"):
        if abs(iters - T64) > 1:
            return False, np.inf, f"T {iters} vs float64 {T64}"
        if iters != T64 and not (t_near_threshold(ref, iters, bw, rel) or t_near_threshold(ref, T64, bw, rel)):
            return False, np.inf, f"T {iters} vs float64 {T64}, shifts {ref['shifts'][max(T64 - 1, 1):T64 + 2]}"
        want = ref["traj"][iters]
        allowed = centre_bound(want, bw)
    else:
        if iters > T64 + 1:
            return False, np.inf, f"reported iterations {iters} > float64 T {T64} + 1"
        want = ref["traj"][T64]
        allowed = centre_bound(want, bw) + DELTA_REL * bw
    err = float(np.linalg.norm(ctr - want))
    ratio = err / allowed
    return ratio <= 1.0, ratio, f"|dc| = {err:.3g} vs {allowed:.3g}"


# ---- Kabsch in float64 ---------------------------------------------------------------------------
def kabsch_f64(A: np.ndarray, B: np.ndarray, reflection_fix: bool = True):
    """least-squares rigid transform A -> B in float64 (basic_utils.py:47-80 with numpy's SVD) -> (R, t, s)"""
    A = np.asarray(A, np.float64)
    B = np.asarray(B, np.float64)
    ca, cb = A.mean(0), B.mean(0)
    H = (A - ca).T @ (B - cb)
    U, s, Vt = np.linalg.svd(H)
    R = Vt.T @ U.T
    if reflection_fix and np.linalg.det(R) < 0:
        Vt[2, :] *= -1
        R = Vt.T @ U.T
    return R, cb - R @ ca, s


def kabsch_residual(A, B, R, t) -> float:
    """sum_i |R a_i + t - b_i|^2 in float64"""
    A = np.asarray(A, np.float64)
    B = np.asarray(B, np.float64)
    return float(((A @ np.asarray(R, np.float64).T + np.asarray(t, np.float64) - B) ** 2).sum())
