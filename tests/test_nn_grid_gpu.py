"""3-NN + inverse-distance weights on per-frame cell grids (pvn3d_three_nn_weights_levels) against oracle/pn2, bit for
bit, at the grid's own edges: points on cell faces, clouds at the per-axis and total cell caps, a 300 m outlier, every
point in one cell, fewer than three finite known points, frames of one batch with very different extents, and known
sets above the grid's size limit (which must take today's kernels, confirmed by the library's launch counter); and the
ball query of both radii on cell grids (pvn3d_ball_query2_levels) against the oracle's ball_query: the four SA levels
in one call, points within ulps of the radius, coincident, NaN / inf points and centres, a far outlier, empty balls,
and centres with more hits than the warp buffer, which take the index-order scan."""
import numpy as np
import pytest

import geo_ref as G
from helpers import t
from oracle import pn2
from pvn3d_b200 import _ext, _lib

pytestmark = pytest.mark.gpu
F32 = np.float32


def _surface(rng, b, n, scale=1.0):
    """depth-like clouds: a wavy sheet of b frames, n points each, in index order of a raster"""
    u = rng.uniform(-0.5, 0.5, (b, n, 2)).astype(F32)
    z = 0.05 * np.sin(6 * u[..., 0]) * np.cos(4 * u[..., 1]) + 0.8
    return (np.concatenate([u, z[..., None]], -1) * scale).astype(F32)


def _sub(rng, x, m):
    """m points of every frame of x (the known set of a level is a subset of the level above)"""
    idx = np.stack([np.sort(rng.choice(x.shape[1], m, replace=False)) for _ in range(x.shape[0])])
    return np.ascontiguousarray(np.take_along_axis(x, idx[..., None].repeat(3, -1), 1))


def _check(cuda_dev, pairs, launches=None):
    """run all pairs in one call; compare every level with the oracle; optionally the number of launches"""
    lib = _lib.load()
    ud, kd = [t(u, cuda_dev) for u, _ in pairs], [t(k, cuda_dev) for _, k in pairs]
    c0 = lib.pvn3d_launch_count()
    got = _ext.three_nn_weights_levels(ud, kd)
    c1 = lib.pvn3d_launch_count()
    if launches is not None:
        assert c1 - c0 == launches, (c1 - c0, launches)
    for lvl, ((u, k), (d2, idx, w)) in enumerate(zip(pairs, got)):
        wd2, widx = pn2.three_nn(u, k)
        gi = idx.cpu().numpy()
        assert np.array_equal(gi, widx), (lvl, u.shape, k.shape, int((gi != widx).sum()))
        assert G.same_bits(d2.cpu().numpy(), wd2), lvl
        assert G.same_bits(w.cpu().numpy(), G.weights_ref(wd2)), lvl
        # the separate ops give the same bits
        sd2, sidx = _ext.three_nn(ud[lvl], kd[lvl])
        assert np.array_equal(sidx.cpu().numpy(), gi), lvl
    return got


def test_pipeline_levels_one_call(cuda_dev):
    """four FP levels of a depth-like batch: one grid-build and one search launch for all of them"""
    rng = np.random.default_rng(0)
    l0 = _surface(rng, 3, 8192)
    l1 = _sub(rng, l0, 2048)
    l2 = _sub(rng, l1, 1024)
    l3 = _sub(rng, l2, 512)
    l4 = _sub(rng, l3, 128)
    _check(cuda_dev, [(l0, l1), (l1, l2), (l2, l3), (l3, l4)], launches=2)


def test_points_on_cell_faces_and_ties(cuda_dev):
    """a lattice of known points, queries on the lattice, on its mid-planes and at its corners: many distances tie
    exactly and many coordinates fall on cell faces; coincident known points tie on the index"""
    g = np.arange(16, dtype=F32) * F32(0.0625)
    lat = np.stack(np.meshgrid(g, g, g[:8], indexing="ij"), -1).reshape(-1, 3)          # 2048 points
    k = np.concatenate([lat, lat[::7]])[None].astype(F32)                             # 2341: coincident pairs
    q = np.concatenate([lat, lat + F32(0.03125), lat[:512] * F32(0.5) + F32(0.03125)])[None].astype(F32)
    _check(cuda_dev, [(np.ascontiguousarray(q), np.ascontiguousarray(k))], launches=2)


def test_cell_caps(cuda_dev):
    """a uniform volume (the total cell cap binds) and a long thin needle (the per-axis cap binds), at the grid's
    largest known set"""
    rng = np.random.default_rng(1)
    vol = rng.uniform(-1, 1, (2, 8192, 3)).astype(F32)
    needle = np.stack([rng.uniform(-50, 50, 8192), rng.uniform(0, 0.01, 8192), rng.uniform(0, 0.01, 8192)], -1)
    needle = needle[None].astype(F32)
    q_vol = rng.uniform(-1.2, 1.2, (2, 4096, 3)).astype(F32)
    q_needle = np.ascontiguousarray(needle[:, ::2] + F32(0.001))
    _check(cuda_dev, [(q_vol, vol)], launches=2)
    _check(cuda_dev, [(q_needle, needle)], launches=2)


def test_far_outlier(cuda_dev):
    """one known point 300 m away makes every cell coarse: slower, never wrong; queries near it and far from all"""
    rng = np.random.default_rng(2)
    x = _surface(rng, 2, 4096)
    k = _sub(rng, x, 1024)
    k[0, 17] = (300.0, -2.0, 0.5)
    k[1, 1000] = (-300.0, 300.0, 300.0)
    q = x.copy()
    q[0, 5] = (299.0, -2.0, 0.5)
    q[1, 7] = (1000.0, 1000.0, -1000.0)
    _check(cuda_dev, [(q, k)], launches=2)


def test_all_points_in_one_cell(cuda_dev):
    """every known point of frame 0 at one position (every distance ties; the index decides), frame 1 in a tiny ball"""
    rng = np.random.default_rng(3)
    k = np.empty((2, 300, 3), F32)
    k[0] = (0.1, 0.2, 0.3)
    k[1] = F32(0.5) + rng.normal(0, 1e-6, (300, 3)).astype(F32)
    q = rng.uniform(-1, 1, (2, 700, 3)).astype(F32)
    q[:, :3] = k[:, :3]
    _check(cuda_dev, [(q, k)], launches=2)


def test_fewer_than_three_finite_known_points(cuda_dev):
    """m = 1 and 2, and m = 5 of which only 2 are finite (NaN and inf are never among the nearest): the empty slots
    hold +inf / 0 and the weights their NaN / 0, as the cascade gives; non-finite queries find nothing"""
    rng = np.random.default_rng(4)
    q = rng.uniform(-1, 1, (2, 257, 3)).astype(F32)
    q[0, 3] = (np.nan, 0, 0)
    q[1, 4] = (np.inf, 0, 0)
    k5 = rng.uniform(-1, 1, (2, 5, 3)).astype(F32)
    k5[:, 0, 1] = np.nan
    k5[:, 2, 0] = np.inf
    k5[:, 4, 2] = -np.inf
    pairs = [(q, np.ascontiguousarray(k5[:, 1:2])), (q, np.ascontiguousarray(k5[:, 1:4:2])), (q, k5)]
    _check(cuda_dev, pairs, launches=2)
    k_none = np.full((2, 4, 3), np.nan, F32)
    _check(cuda_dev, [(q, k_none)], launches=2)


def test_frames_with_very_different_extents(cuda_dev):
    """one grid per frame: a 1 mm, a 1 m and a 100 m frame in one batch"""
    rng = np.random.default_rng(5)
    x = np.concatenate([_surface(rng, 1, 4096, s) for s in (1e-3, 1.0, 100.0)])
    k = _sub(rng, x, 1024)
    _check(cuda_dev, [(x, k)], launches=2)


def test_known_sets_above_the_grid_limit_take_todays_kernels(cuda_dev):
    """m = 8193 is above the grid's limit: that level runs three_nn (exhaustive scan, one launch) and the weights
    kernel, the other level the grid (two launches)"""
    rng = np.random.default_rng(6)
    lib = _lib.load()
    assert lib.pvn3d_three_nn_grid_supported(4096, 8192) and not lib.pvn3d_three_nn_grid_supported(4096, 8193)
    big = rng.uniform(-1, 1, (1, 8193, 3)).astype(F32)
    q = rng.uniform(-1, 1, (1, 2048, 3)).astype(F32)
    small = _sub(rng, q, 512)
    _check(cuda_dev, [(q, big), (q, small)], launches=2 + 2)


# ---- ball query of both radii on cell grids (pvn3d_ball_query2_levels) ---------------------------------------------
def _check_ball(cuda_dev, levels, launches=None):
    """levels: [(cloud, centres, (r0, r1), (ns0, ns1))], run in one call, each radius against the oracle"""
    lib = _lib.load()
    cl, ce = [t(x, cuda_dev) for x, _, _, _ in levels], [t(c, cuda_dev) for _, c, _, _ in levels]
    c0 = lib.pvn3d_launch_count()
    got = _ext.ball_query2_levels(ce, cl, [r for _, _, r, _ in levels], [ns for _, _, _, ns in levels])
    c1 = lib.pvn3d_launch_count()
    if launches is not None:
        assert c1 - c0 == launches, (c1 - c0, launches)
    for lvl, ((x, c, radii, nss), pair) in enumerate(zip(levels, got)):
        for s in range(2):
            want = pn2.ball_query(c, x, float(F32(radii[s])), nss[s])
            g = pair[s].cpu().numpy()
            assert np.array_equal(g, want), (lvl, s, x.shape, int((g != want).sum()))


def test_ball_pipeline_levels_one_call(cuda_dev):
    """the four SA levels of a depth-like batch: one grid-build and one search launch for all of them"""
    rng = np.random.default_rng(10)
    l0 = _surface(rng, 3, 12288)
    l1 = _sub(rng, l0, 2048)
    l2 = _sub(rng, l1, 1024)
    l3 = _sub(rng, l2, 512)
    l4 = _sub(rng, l3, 128)
    spec = [((0.0175, 0.025), (16, 32)), ((0.025, 0.05), (16, 32)), ((0.05, 0.1), (16, 32)), ((0.1, 0.2), (16, 32))]
    _check_ball(cuda_dev, [(x, c, r, ns) for (x, c), (r, ns) in zip([(l0, l1), (l1, l2), (l2, l3), (l3, l4)], spec)],
                launches=2)


def test_ball_edges(cuda_dev):
    """points within ulps of the radius on every axis, coincident points, NaN / inf points and centres, a 300 m outlier,
    empty balls, radii larger-first and equal"""
    rng = np.random.default_rng(11)
    x = _surface(rng, 2, 4096)
    c = _sub(rng, x, 512)
    r = F32(0.05)
    for i in range(40):                       # shell points around centre i of frame 0, on the axes and diagonals
        d = np.zeros(3, F32)
        d[i % 3] = np.nextafter(r, F32(0) if i % 2 else F32(1)) * (1 if i % 4 < 2 else -1)
        x[0, 100 + i] = c[0, i] + d
    x[1, 10:30] = x[1, 5]                     # coincident points
    x[0, 7] = (np.nan, 0, 0)
    x[1, 8] = (np.inf, 0.5, 0.5)
    x[1, 9] = (300.0, -300.0, 300.0)
    c[0, 500] = (np.nan, 0, 0)
    c[1, 501] = (-np.inf, 0, 0)
    c[1, 502] = (5.0, 5.0, 5.0)               # empty ball
    _check_ball(cuda_dev, [(x, c, (0.05, 0.025), (16, 32)), (x, c, (0.05, 0.05), (32, 16))], launches=2)


def test_ball_overflowing_buffer_scans_in_index_order(cuda_dev):
    """a cluster of 3000 points inside both balls of some centres: more hits than the warp buffer (512) holds, so those
    centres take the index-order scan; the cluster is interleaved in index order with far points"""
    rng = np.random.default_rng(12)
    far = rng.uniform(-1, 1, (1, 6000, 3)).astype(F32)
    blob = (rng.normal(0, 0.004, (1, 3000, 3)) + 0.2).astype(F32)
    x = np.empty((1, 9000, 3), F32)
    x[:, 0::3], x[:, 1::3], x[:, 2::3] = far[:, :3000], blob, far[:, 3000:]
    c = np.concatenate([blob[:, :64], far[:, :64]], 1)
    assert _lib.load().pvn3d_ball_grid_supported(9000, 128, 256, 256)
    assert not _lib.load().pvn3d_ball_grid_supported(9000, 128, 257, 16)
    _check_ball(cuda_dev, [(x, np.ascontiguousarray(c), (0.02, 0.04), (256, 64))], launches=2)
