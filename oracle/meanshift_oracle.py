"""TEST INFRASTRUCTURE -- CPU restatement (torch float32 ops) of the reference's vote clustering.

Follows pvn3d/lib/utils/meanshift_pytorch.py:13-51 op for op on CPU tensors, so every rounding
the reference performs is reproduced by the same torch CPU kernels:
  * gaussian_kernel (:13-15): (1/(bw*sqrt(2*float32(pi)))) * exp(-0.5*(dis/bw)**2)
  * fit (:24-51): all points are seeds; C <- sum_j w_ij A_j / sum_j w_ij until
    max_i |dC_i| < bw*1e-3 or it > max_iter; the densest INPUT point (count of |A_i-A_j| < bw,
    first index on ties) selects the returned seed and the labels.
Pinned against the real class (imported from /root/reference) by tests/golden/make_golden_cpu.py:
identical bits for (ctr, labels, iterations) on every recorded case; the recorded outputs are
committed as tests/golden/ms_*.npz.

Also the timed CPU baseline of bench.py (cpu_baseline / --impl reference), because the reference's
own "CPU MeanShift" is exactly this code path on CPU tensors (SURVEY section 0).
"""
from __future__ import annotations

import math

import numpy as np
import torch


def gaussian_kernel(distance: torch.Tensor, bandwidth: float) -> torch.Tensor:
    # meanshift_pytorch.py:13-15 -- coefficient is a float32 0-dim tensor
    coef = 1 / (bandwidth * torch.sqrt(2 * torch.tensor(np.pi)))
    return coef * torch.exp(-0.5 * (distance / bandwidth) ** 2)


class MeanShiftOracle:
    def __init__(self, bandwidth: float = 0.05, max_iter: int = 300):
        self.bandwidth = bandwidth
        self.stop_thresh = bandwidth * 1e-3  # :21
        self.max_iter = max_iter
        self.n_iter = 0

    def fit(self, A: torch.Tensor):
        """A [N,3] float32 CPU -> (C[max_idx] [3], labels [N] bool)"""
        assert A.device.type == "cpu" and A.dtype == torch.float32
        n, c = A.shape
        pts = A.reshape(1, n, c).expand(n, n, c)               # Ar: row i = all points (:33)
        C = A.clone()                                          # (:31)
        it = 0
        while True:
            it += 1
            seeds = C.reshape(n, 1, c).expand(n, n, c)         # Cr (:34)
            dis = torch.norm(seeds - pts, dim=2)               # (:35)
            w = gaussian_kernel(dis, self.bandwidth).reshape(n, n, 1)
            new_C = torch.sum(w * pts, dim=1) / torch.sum(w, dim=1)   # (:37)
            shift = torch.norm(new_C - C, dim=1)               # (:39)
            C = new_C
            if torch.max(shift) < self.stop_thresh or it > self.max_iter:   # (:42)
                break
        self.n_iter = it
        _, max_idx, labels = density_labels(A, self.bandwidth)
        return C[max_idx, :], labels


def density_labels(A: torch.Tensor, bandwidth: float):
    """The exact part of fit (:46-50) on A [N,3] float32 CPU -> (num_in [N] int64, max_idx 0-dim int64,
    labels [N] bool).  It depends on the input points alone, never on the iterations."""
    n, c = A.shape
    pts = A.reshape(1, n, c).expand(n, n, c)                   # Ar (:33)
    own = A.reshape(n, 1, c).expand(n, n, c)                   # Cr rebuilt from the INPUTS (:46)
    dis = torch.norm(pts - own, dim=2)                         # (:47)
    num_in = torch.sum(dis < bandwidth, dim=1)                 # (:48)
    _, max_idx = torch.max(num_in, 0)                          # first maximal index on CPU (:49)
    labels = dis[max_idx] < bandwidth                          # (:50)
    return num_in, max_idx, labels


def best_fit_transform(A: np.ndarray, B: np.ndarray) -> np.ndarray:
    """pvn3d/lib/utils/basic_utils.py:47-80 (Kabsch with reflection fix); float32 inputs keep the
    reference's float32 LAPACK path; returns a float64 3x4."""
    assert A.shape == B.shape
    m = A.shape[1]
    ca, cb = np.mean(A, axis=0), np.mean(B, axis=0)
    H = np.dot((A - ca).T, B - cb)
    U, _, Vt = np.linalg.svd(H)
    R = np.dot(Vt.T, U.T)
    if np.linalg.det(R) < 0:
        Vt[m - 1, :] *= -1
        R = np.dot(Vt.T, U.T)
    t = cb.T - np.dot(R, ca.T)
    T = np.zeros((3, 4))
    T[:, :3] = R
    T[:, 3] = t
    return T
