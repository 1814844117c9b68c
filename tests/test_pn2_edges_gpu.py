"""Every coordinate-only kernel of hot path A at the edges of its own dispatch, bit for bit against oracle/pn2 (the
index ops) or the numpy restatements of tests/geo_ref.py (weights, factor table, centre term).

Inputs and the mutants each case must reject are in tests/pn2_edge_cases.py.  Which path a case takes follows from
its shape (fps.cu: launch_regs<PPT> for ceil(n / 512) <= PPT, the generic kernel above 12288 points; query_group.cu:
256-point boxes above 131072 points, CW = 4 / 2 / 1 centres per warp for ns0 + ns1 <= 64 / 128 / 256; pn2_ops.cu: the
x-sorted walk for 512 <= m <= 4096 and n >= 2 m) and, for 3-NN, is confirmed by the library's launch counter: the
walk is two launches (sort + walk), the exhaustive scan one.
"""
import numpy as np
import pytest
import torch

import geo_ref as G
import pn2_edge_cases as C
from helpers import t
from oracle import pn2
from pvn3d_b200 import _ext, _lib, mlp

pytestmark = pytest.mark.gpu
F32 = np.float32


def _reject(names, build_mutants, inputs, refs, flat=lambda r: r):
    for nm, mu in build_mutants(names, inputs, refs).items():
        assert C.some_differ([flat(r) for r in refs], mu), f"the inputs cannot tell the oracle from mutant {nm!r}"


@pytest.mark.parametrize("name", list(C.FPS_CASES))
def test_fps_edges(cuda_dev, name):
    build, names = C.FPS_CASES[name]
    inputs = build()
    refs = [pn2.furthest_point_sampling(x, m) for x, m in inputs]
    for (x, m), want in zip(inputs, refs):
        got = _ext.furthest_point_sampling(t(x, cuda_dev), m).cpu().numpy()
        assert np.array_equal(got, want), (name, x.shape, m, int((got != want).sum()))
    _reject(names, C.fps_mutants, inputs, refs)


@pytest.mark.parametrize("name", list(C.BALL_CASES))
def test_ball_query_edges(cuda_dev, name):
    build, names = C.BALL_CASES[name]
    inputs = build()
    refs = C.ball_refs(inputs)
    for (x, c, radii, nss), want in zip(inputs, refs):
        xd, cd = t(x, cuda_dev), t(c, cuda_dev)
        got = _ext.ball_query2(cd, xd, radii, nss)
        for s in range(2):
            g = got[s].cpu().numpy()
            assert np.array_equal(g, want[s]), (name, x.shape, radii, nss, s, int((g != want[s]).sum()))
            assert g.min() >= 0 and g.max() < x.shape[1]
            one = _ext.ball_query(cd, xd, radii[s], nss[s]).cpu().numpy()           # the single-radius op
            assert np.array_equal(one, want[s]), (name, "ball_query", s)
        if x.shape[1] <= 12288:                                                     # idx of the grouping form
            _, gi = _ext.query_and_group2(xd, cd, None, radii, nss)
            assert all(np.array_equal(gi[s].cpu().numpy(), want[s]) for s in range(2)), (name, "query_and_group2")
    _reject(names, C.ball_mutants, inputs, refs)


def test_ball_query2_refuses_more_than_256_slots_per_centre(cuda_dev):
    x = G.uniform_cloud(1, 4096, 66, 0.0, 0.4)
    xd, cd = t(x, cuda_dev), t(C._strided_centres(x, 64), cuda_dev)
    i0 = torch.full((1, 64, 129), -7, dtype=torch.int32, device=cuda_dev)
    i1 = torch.full((1, 64, 128), -7, dtype=torch.int32, device=cuda_dev)
    lib = _lib.load()
    with torch.cuda.device(cuda_dev):
        rc = lib.pvn3d_query_and_group2(xd.data_ptr(), cd.data_ptr(), 0, 0, 1, 4096, 64, 0, 0.04, 129, i0.data_ptr(), 0,
                                        0.08, 128, i1.data_ptr(), 0, torch.cuda.current_stream(cuda_dev).cuda_stream)
    torch.cuda.synchronize()
    assert rc == -2                                                    # PVN3D_ERR_UNSUPPORTED
    assert bool((i0 == -7).all()) and bool((i1 == -7).all())          # outputs untouched
    with pytest.raises(_lib.Pvn3dError, match="unsupported size"):
        _ext.ball_query2(cd, xd, (0.04, 0.08), (129, 128))


@pytest.mark.parametrize("name", list(C.NN_CASES))
def test_three_nn_edges(cuda_dev, name):
    build, names = C.NN_CASES[name]
    inputs = build()
    refs = [pn2.three_nn(u, k) for u, k in inputs]
    lib = _lib.load()
    for (u, k), (wd2, widx) in zip(inputs, refs):
        before = lib.pvn3d_launch_count()
        d2, idx = _ext.three_nn(t(u, cuda_dev), t(k, cuda_dev))
        assert lib.pvn3d_launch_count() - before == (2 if C.nn_takes_slab(k.shape[1], u.shape[1]) else 1)
        idx, d2 = idx.cpu().numpy(), d2.cpu().numpy()
        assert np.array_equal(idx, widx), (name, u.shape, k.shape, int((idx != widx).sum()))
        assert G.same_bits(d2, wd2), (name, u.shape, k.shape)
        # and the weights the engine derives from them
        w = mlp.three_nn_weights(t(wd2, cuda_dev)).cpu().numpy()
        assert G.same_bits(w, G.weights_ref(wd2)), (name, "weights")
    _reject(names, C.nn_mutants, inputs, refs, flat=lambda r: r[1])


@pytest.mark.parametrize("rows", [393216, 1000, 3])          # 32 x 12288 (the benchmark's FP1), not a multiple of 256
def test_three_nn_weights_bit_exact(cuda_dev, rows):
    d2 = C.weight_inputs(rows, rows)
    got = mlp.three_nn_weights(t(d2, cuda_dev)).cpu().numpy()
    want = G.weights_ref(d2)
    assert G.same_bits(got, want), int((G.bits(got) != G.bits(want)).sum())
    assert G.weights_err_over_bound(got, G.weights_f64(d2)) <= 1.0
    assert not G.same_bits(G.mut_weights_no_eps(d2), want)


@pytest.mark.parametrize("rows,c_feat,scale", [(393216, 6, "raster"), (4099, 0, "raster"), (4099, 96, "far"),
                                               (1001, 512, "tiny"), (300, 6, "far"), (300, 6, "tiny")])
def test_sa_factor_table_bit_exact(cuda_dev, rows, c_feat, scale):
    rng = np.random.default_rng(rows + c_feat)
    b = 32 if rows == 393216 else 1
    xyz = G.raster_cloud(b, rows // b, 90) if rows % 12288 == 0 else G.uniform_cloud(1, rows, 91, -1.0, 1.0)
    xyz = {"raster": xyz, "far": G.far(xyz), "tiny": G.tiny(xyz)}[scale]
    ldf = c_feat + 3                                                   # rows wider than the descriptors
    feat = rng.normal(size=(rows, ldf)).astype(np.float32) if c_feat else None
    k_pad = (c_feat + 6 + 31) // 32 * 32
    fd = t(feat, cuda_dev) if c_feat else None
    got = mlp.sa_factor_table(t(xyz, cuda_dev), fd.data_ptr() if c_feat else 0, ldf, c_feat, k_pad).cpu().numpy()
    want = G.factor_table_ref(xyz.reshape(-1, 3), feat, c_feat, k_pad)
    assert np.array_equal(G.bits(got), G.bits(want)), int((G.bits(got) != G.bits(want)).sum())
    assert G.split_rel_err(xyz.reshape(-1, 3), got, c_feat) <= 2.0 ** -21
    assert not np.array_equal(G.bits(G.mut_table_no_lo(want, c_feat)), G.bits(want))


@pytest.mark.parametrize("rows,n_pad,scale", [(65536, 32, "raster"), (1001, 64, "far"), (1001, 128, "tiny"), (7, 16, "raster")])
def test_sa_centre_term_against_float64(cuda_dev, rows, n_pad, scale):
    rng = np.random.default_rng(rows + n_pad)
    c = G.uniform_cloud(1, rows, 92, -1.0, 1.0)
    c = {"raster": c, "far": G.far(c), "tiny": G.tiny(c)}[scale]
    wx = G.tf32(rng.normal(size=(n_pad, 3)).astype(np.float32))
    bias = rng.normal(size=(n_pad,)).astype(np.float32)
    got = mlp.sa_centre_term(t(c, cuda_dev), t(wx, cuda_dev), t(bias, cuda_dev)).cpu().numpy().astype(np.float64)
    want, bound = G.centre_term_f64(c[0], wx, bias)
    worst = float((np.abs(got - want) / bound).max())
    print(f"sa_centre_term rows={rows} n_pad={n_pad} {scale}: worst |got - ref| / bound = {worst:.3f}")
    assert worst <= 1.0
    wrong, _ = G.centre_term_f64(c[0], wx, -bias)                      # V = Wx c + b: the sign of the bias flipped
    assert float((np.abs(wrong - want) / bound).max()) > 1e3


@pytest.mark.parametrize("b,n,m,c", [(32, 2048, 1024, 9), (3, 1001, 37, 5), (1, 49152, 2048, 131)])
def test_gather_and_transposes_bit_exact(cuda_dev, b, n, m, c):
    rng = np.random.default_rng(n + m)
    xyz = rng.normal(size=(b, n, 3)).astype(np.float32)
    idx = rng.integers(0, n, size=(b, m)).astype(np.int32)
    got = _ext.gather_xyz(t(xyz, cuda_dev), t(idx, cuda_dev)).cpu().numpy()
    assert np.array_equal(got, G.gather_rows(xyz, idx))
    assert not np.array_equal(got, G.mut_frame0(G.gather_rows(xyz, idx))) or b == 1
    f = rng.normal(size=(b, c, n)).astype(np.float32)
    nc = _ext.transpose_cn_to_nc(t(f, cuda_dev))
    assert np.array_equal(nc.cpu().numpy(), f.transpose(0, 2, 1))
    assert np.array_equal(_ext.transpose_nc_to_cn(nc).cpu().numpy(), f)
