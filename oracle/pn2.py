"""TEST INFRASTRUCTURE -- numpy front-end of libpn2_oracle.so (oracle/pn2_oracle.c).

Each function takes/returns C-contiguous numpy arrays with the dtypes and layouts of the reference
ops (pvn3d/_ext-src/include/*.h).  Batches are split across Python threads (ctypes drops the GIL;
this image has no libgomp), `threads=None` -> os.cpu_count().
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libpn2_oracle.so")
_lib = None


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "pn2_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.run(["make", "-C", _HERE, "libpn2_oracle.so"] + (["-B"] if force else []), check=True,
                       capture_output=True)
    return _SO


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(_SO)
    return _lib


def _f(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a, a.ctypes.data_as(ctypes.c_void_p)


def _i(a):
    a = np.ascontiguousarray(a, dtype=np.int32)
    return a, a.ctypes.data_as(ctypes.c_void_p)


def _over_batch(b, fn, threads=None):
    nt = min(b, threads or os.cpu_count() or 1)
    if nt <= 1:
        for i in range(b):
            fn(i)
        return
    with ThreadPoolExecutor(max_workers=nt) as ex:
        list(ex.map(fn, range(b)))


def opt_n_threads(n: int) -> int:
    return int(lib().oracle_opt_n_threads(ctypes.c_int(n)))


def sqdist(q, pts):
    """q [nq,3], pts [n,3] -> [nq,n] f32: the squared distance of the ops below, bit for bit (oracle_sqdist)"""
    q, qp = _f(q); pts, pp = _f(pts)
    out = np.zeros((q.shape[0], pts.shape[0]), np.float32)
    lib().oracle_sqdist(qp, q.shape[0], pp, pts.shape[0], out.ctypes.data_as(ctypes.c_void_p))
    return out


def furthest_point_sampling(xyz, m, threads=None):
    xyz, _ = _f(xyz)
    b, n, _3 = xyz.shape
    out = np.zeros((b, m), np.int32)
    L = lib()

    def one(i):
        L.oracle_furthest_point_sampling(xyz[i].ctypes.data_as(ctypes.c_void_p), 1, n, m,
                                         out[i].ctypes.data_as(ctypes.c_void_p))
    _over_batch(b, one, threads)
    return out


def gather_points(points, idx):
    points, pp = _f(points); idx, ip = _i(idx)
    b, c, n = points.shape; m = idx.shape[1]
    out = np.zeros((b, c, m), np.float32)
    lib().oracle_gather_points(pp, ip, b, c, n, m, out.ctypes.data_as(ctypes.c_void_p))
    return out


def gather_points_grad(grad_out, idx, n):
    grad_out, gp = _f(grad_out); idx, ip = _i(idx)
    b, c, m = grad_out.shape
    out = np.zeros((b, c, n), np.float32)
    lib().oracle_gather_points_grad(gp, ip, b, c, n, m, out.ctypes.data_as(ctypes.c_void_p))
    return out


def ball_query(new_xyz, xyz, radius, nsample, threads=None):
    new_xyz, _ = _f(new_xyz); xyz, _ = _f(xyz)
    b, n, _3 = xyz.shape; m = new_xyz.shape[1]
    out = np.zeros((b, m, nsample), np.int32)
    L = lib()

    def one(i):
        L.oracle_ball_query(new_xyz[i].ctypes.data_as(ctypes.c_void_p), xyz[i].ctypes.data_as(ctypes.c_void_p),
                            1, n, m, ctypes.c_float(radius), nsample, out[i].ctypes.data_as(ctypes.c_void_p))
    _over_batch(b, one, threads)
    return out


def group_points(points, idx):
    points, pp = _f(points); idx, ip = _i(idx)
    b, c, n = points.shape; _, m, s = idx.shape
    out = np.zeros((b, c, m, s), np.float32)
    lib().oracle_group_points(pp, ip, b, c, n, m, s, out.ctypes.data_as(ctypes.c_void_p))
    return out


def group_points_grad(grad_out, idx, n):
    grad_out, gp = _f(grad_out); idx, ip = _i(idx)
    b, c, m, s = grad_out.shape
    out = np.zeros((b, c, n), np.float32)
    lib().oracle_group_points_grad(gp, ip, b, c, n, m, s, out.ctypes.data_as(ctypes.c_void_p))
    return out


def three_nn(unknown, known, threads=None):
    unknown, _ = _f(unknown); known, _ = _f(known)
    b, n, _3 = unknown.shape; m = known.shape[1]
    d = np.zeros((b, n, 3), np.float32); ix = np.zeros((b, n, 3), np.int32)
    L = lib()

    def one(i):
        L.oracle_three_nn(unknown[i].ctypes.data_as(ctypes.c_void_p), known[i].ctypes.data_as(ctypes.c_void_p),
                          1, n, m, d[i].ctypes.data_as(ctypes.c_void_p), ix[i].ctypes.data_as(ctypes.c_void_p))
    _over_batch(b, one, threads)
    return d, ix


def three_interpolate(points, idx, weight):
    points, pp = _f(points); idx, ip = _i(idx); weight, wp = _f(weight)
    b, c, m = points.shape; n = idx.shape[1]
    out = np.zeros((b, c, n), np.float32)
    lib().oracle_three_interpolate(pp, ip, wp, b, c, m, n, out.ctypes.data_as(ctypes.c_void_p))
    return out


def three_interpolate_grad(grad_out, idx, weight, m):
    grad_out, gp = _f(grad_out); idx, ip = _i(idx); weight, wp = _f(weight)
    b, c, n = grad_out.shape
    out = np.zeros((b, c, m), np.float32)
    lib().oracle_three_interpolate_grad(gp, ip, wp, b, c, n, m, out.ctypes.data_as(ctypes.c_void_p))
    return out


def query_and_group(xyz, new_xyz, features, radius, nsample, threads=None):
    """features channel-major [B,C,N] or None; returns (out [B,3+C,M,S], idx [B,M,S])"""
    xyz, _ = _f(xyz); new_xyz, _ = _f(new_xyz)
    b, n, _3 = xyz.shape; m = new_xyz.shape[1]
    c = 0 if features is None else features.shape[1]
    feats = np.zeros((b, 0, n), np.float32) if features is None else _f(features)[0]
    out = np.zeros((b, 3 + c, m, nsample), np.float32)
    idx = np.zeros((b, m, nsample), np.int32)
    L = lib()

    def one(i):
        L.oracle_query_and_group(xyz[i].ctypes.data_as(ctypes.c_void_p), new_xyz[i].ctypes.data_as(ctypes.c_void_p),
                                 feats[i].ctypes.data_as(ctypes.c_void_p), 1, n, m, c, ctypes.c_float(radius),
                                 nsample, idx[i].ctypes.data_as(ctypes.c_void_p), out[i].ctypes.data_as(ctypes.c_void_p))
    _over_batch(b, one, threads)
    return out, idx
