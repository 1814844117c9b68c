"""The inputs of tests/test_pn2_edges_gpu.py: every coordinate kernel at the edges of its own dispatch.

A case is a list of inputs plus the names of the mutants (tests/geo_ref.py) it must tell from the oracle: the kernel
has to equal the oracle on every input of the case, and every named mutant has to differ from the oracle on at least
one of them.  The second half needs no GPU and is also run by tests/test_geo_ref_host.py.
"""
import numpy as np

import geo_ref as G
from oracle import pn2

F32 = np.float32


def _tie_cloud(b, n, seed):
    """lattice points away from the origin with coincident groups: exact ties in every arg-max and cascade"""
    return G.with_duplicates(G.lattice(b, n, 0.01, seed, 0, 40, offset=0.3), seed + 1)


# ---- furthest-point sampling: inputs are (xyz [B,n,3], m) -------------------------------------------------------
def _fps_regs(p):
    # n = 512 p is the last cloud launch_regs<p> takes, 512 p + 1 the first of the next instantiation (p = 24: the
    # generic kernel, min-distances in global memory)
    return [(_tie_cloud(2, 512 * p, p), 33), (_tie_cloud(2, 512 * p + 1, 100 + p), 33)]


def _fps_pow2():
    # the reference block size 2^floor(log2 n) feeds the tie-break: both sides of every power of two up to 512
    return [(_tie_cloud(2, n, 200 + n), min(n, 8)) for n in
            (1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 37, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 513)]


def _fps_small_xyz(n, seed, at0):
    x = G.with_duplicates(G.uniform_cloud(2, n, seed), seed + 1)
    x[:, 5::7] *= F32(0.01)                          # |p|^2 <= 3e-4: never chosen
    if at0:
        x[:, 0] = [0.01, 0.0, 0.02]                  # the start point itself is ineligible but is still out[0]
    return x


FPS_CASES = {
    **{f"regs{p}": (lambda p=p: _fps_regs(p), ["lowest_index", "frame0"]) for p in (1, 2, 4, 8, 12, 16, 24)},
    "pow2_sides": (_fps_pow2, ["frame0"]),
    "generic_ragged": (lambda: [(_tie_cloud(2, 49000, 7), 64)], ["lowest_index", "frame0"]),
    "m_is_1": (lambda: [(_tie_cloud(2, 1000, 8), 1), (_tie_cloud(1, 13000, 9), 1)], []),
    # m = n: every eligible point is taken, then the oracle keeps choosing among points at distance 0
    "m_is_n": (lambda: [(_fps_small_xyz(700, 10, False), 700), (_fps_small_xyz(12289, 11, True)[:1], 12289)],
               ["lowest_index"]),
    "ineligible": (lambda: [(_fps_small_xyz(3000, 12, True), 257), (_fps_small_xyz(13000, 13, True), 130)],
                   ["no_skip", "frame0"]),
    "all_ineligible": (lambda: [(G.tiny(G.uniform_cloud(2, 600, 14), 0.01), 9),
                                (G.tiny(G.uniform_cloud(2, 12800, 15), 0.01), 9)], ["no_skip"]),
    "batch32": (lambda: [(_tie_cloud(32, 2048, 16), 64)], ["frame0", "lowest_index"]),
    "bench_stress": (lambda: [(G.with_duplicates(G.uniform_cloud(8, 49152, 17), 18), 2048)], ["frame0", "lowest_index"]),
}


def fps_mutants(names, inputs, refs):
    out = {}
    for nm in names:
        if nm == "frame0":
            out[nm] = [G.mut_frame0(r) for r in refs]
        else:   # the numpy sampler is serial: frame 0 only, the other frames keep the oracle's answer
            res = []
            for (xyz, m), r in zip(inputs, refs):
                mu = r.copy()
                mu[0] = G.fps_lowest_index(xyz[0], m, skip=nm != "no_skip")
                res.append(mu)
            out[nm] = res
    return out


# ---- ball query: inputs are (cloud [B,n,3], centres [B,m,3], radii, nsamples) ----------------------------------
def _strided_centres(x, m):
    return np.ascontiguousarray(x[:, :: max(1, x.shape[1] // m)][:, :m])


def _ball_orders():
    x = G.raster_cloud(2, 12288, 30)
    res = []
    for y in (x, G.sorted_cloud(x, 0), G.sorted_cloud(x, 1), G.sorted_cloud(x, 2), G.shuffled(x, 31)):
        res.append((y, _strided_centres(y, 512), (0.0175, 0.025), (16, 32)))
    return res


def _ball_big(n):
    x = G.sorted_cloud(G.uniform_cloud(1, n, n, 0.0, 1.0), 0)
    return [(x, _strided_centres(x, 300), (0.01, 0.02), (16, 32))]


def _ball_tails():
    res = []
    for n in (1280, 1281, 1407, 20):
        x = G.uniform_cloud(2, n, 40 + n, 0.0, 0.3)
        res.append((x, _strided_centres(x, max(5, n // 8)), (0.025, 0.05), (16, 32)))
    return res


def _ball_shell(radii):
    cloud, centres, _ = G.radius_shell(12288, 256, radii, 50)
    return [(cloud, centres, radii, (16, 32))]


def _ball_ns():
    x = G.uniform_cloud(2, 4096, 60, 0.0, 0.4)
    c = _strided_centres(x, 300)
    return [(x, c, (0.04, 0.08), nss) for nss in ((32, 32), (33, 32), (64, 32), (100, 100))]   # CW 4, 2, 2, 1


def _ball_fill():
    x = G.uniform_cloud(2, 4096, 61, 0.0, 0.4)
    x[:, :40] = x[:, :1]                             # 40 coincident points first: full inside the first 32-point step
    c = _strided_centres(x, 200)
    c[:, 1] = 9.0                                    # empty ball
    return [(x, c, (0.004, 0.2), (16, 32))]          # the small radius never fills, the large one fills at once


def _ball_y():
    rng = np.random.default_rng(62)
    x = G.uniform_cloud(2, 4096, 63, 0.0, 0.4)
    c = _strided_centres(x, 256)
    c[..., 1] = F32(0.2)                             # every centre in one y bucket
    cw = rng.uniform(-5e5, 5e5, size=(2, 256, 3)).astype(np.float32)        # y spread over 1e6 m
    xw = (np.repeat(cw, 8, 1) + rng.uniform(-0.06, 0.06, size=(2, 2048, 3)).astype(np.float32)).astype(np.float32)
    return [(x, c, (0.025, 0.05), (16, 32)), (xw, cw, (0.05, 0.1), (16, 32))]


def _ball_scales():
    x = G.raster_cloud(2, 4096, 64)
    xf, xt = G.far(x), G.tiny(x)
    return [(xf, _strided_centres(xf, 256), (0.025, 0.05), (16, 32)),
            (xt, _strided_centres(xt, 256), (0.025e-4, 0.05e-4), (16, 32))]


def _ball_nonfinite():
    x = G.uniform_cloud(2, 4096, 65, 0.0, 0.4)
    c = _strided_centres(x, 256)
    x[0, 100, 0], x[0, 200, 1], x[0, 300, 2], x[1, 4095, 0] = np.nan, np.inf, -np.inf, np.nan
    c[0, 3, 0], c[0, 4, 1], c[0, 5, 2], c[1, 255, 1] = np.nan, np.inf, -np.inf, np.nan
    return [(x, c, (0.025, 0.05), (16, 32))]


BALL_CASES = {
    "orders_12288": (_ball_orders, ["pad_zero", "scan_order", "frame0"]),
    "raster_49152": (lambda: [(lambda x: (x, _strided_centres(x, 2048), (0.0175, 0.025), (16, 32)))(G.raster_cloud(2, 49152, 32))],
                     ["pad_zero", "scan_order", "frame0"]),
    "n_131072": (lambda: _ball_big(131072), ["pad_zero", "scan_order"]),          # 1024 boxes of 128
    "n_131273_blk256": (lambda: _ball_big(131273), ["pad_zero", "scan_order"]),   # 513 boxes of 256
    "tails": (_ball_tails, ["pad_zero", "scan_order", "frame0"]),
    "shell": (lambda: _ball_shell((0.0175, 0.025)), ["le", "pad_zero", "scan_order"]),
    "shell_larger_first": (lambda: _ball_shell((0.025, 0.0175)), ["le", "pad_zero"]),
    "shell_equal": (lambda: _ball_shell((0.025, 0.025)), ["le", "pad_zero"]),
    "ns_sums": (_ball_ns, ["pad_zero", "scan_order", "frame0"]),
    "fill": (_ball_fill, ["pad_zero", "scan_order", "frame0"]),
    "centre_y": (_ball_y, ["pad_zero", "scan_order", "frame0"]),
    "far_tiny": (_ball_scales, ["pad_zero", "scan_order", "frame0"]),
    "nonfinite": (_ball_nonfinite, ["pad_zero", "scan_order", "frame0"]),
}


def ball_refs(inputs):
    """per input: [idx of radius 0, idx of radius 1]"""
    return [[pn2.ball_query(c, x, float(F32(r)), ns) for r, ns in zip(radii, nss)] for x, c, radii, nss in inputs]


def ball_mutants(names, inputs, refs):
    out = {}
    for nm in names:
        res = []
        for (x, c, radii, nss), ref in zip(inputs, refs):
            if nm == "pad_zero":
                res.append([G.mut_ball_pad_zero(r) for r in ref])
            elif nm == "scan_order":
                res.append([G.mut_ball_scan_order(r, c) for r in ref])
            elif nm == "frame0":
                res.append([G.mut_frame0(r) for r in ref])
            elif nm == "le":
                res.append([G.mut_ball_le(r, c, x, float(F32(rad)), np.arange(6)) for r, rad in zip(ref, radii)])
        out[nm] = res
    return out


# ---- 3-NN: inputs are (unknown [B,n,3], known [B,m,3]) ---------------------------------------------------------
def nn_takes_slab(m, n):
    return 512 <= m <= 4096 and n >= 2 * m


def _nn_pair(b, m, n, seed):
    known = _tie_cloud(b, m, seed)
    unk = G.lattice(b, n, 0.01, seed + 2, -5, 45, offset=0.3)      # a wider grid: queries outside the x range too
    unk[:, : max(1, m // 8)] = known[:, : max(1, m // 8)]           # queries ON known points
    return unk, known


def _nn_shared(cols):
    unk, known = _nn_pair(2, 1024, 2500, 70 + len(cols))
    known[..., cols] = F32(0.45)
    return [(unk, known)]


def _nn_zero_x():
    unk, known = _nn_pair(2, 600, 1300, 75)
    known[:, ::2, 0] = F32(0.0)
    known[:, 1::4, 0] = F32(-0.0)
    unk[:, ::3, 0] = F32(-0.0)
    return [(unk, known)]


def _nn_bench():
    x = G.raster_cloud(2, 49152, 76)
    return [(x, np.ascontiguousarray(x[:, ::24]))]                  # every known point is also a query


def _nn_nonfinite():
    unk, known = _nn_pair(2, 600, 1300, 77)
    known[0, 5, 0], known[0, 300, 0], known[1, 7, 1], known[1, 9, 0], known[1, 11, 0] = np.nan, np.nan, np.nan, np.inf, -np.inf
    return [(unk, known)]


NN_CASES = {
    "slab_rule": (lambda: [_nn_pair(2, m, n, m + n) for m, n in
                           ((511, 4096), (512, 1023), (512, 1024), (4096, 8192), (4097, 9000), (1024, 2048))],
                  ["last_index", "ties_unordered", "frame0"]),
    "bench_49152x2048": (_nn_bench, ["frame0"]),
    "tiny_m": (lambda: [_nn_pair(2, m, 100, 80 + m) for m in (1, 2, 3)], ["frame0"]),
    "slab_not_pow2": (lambda: [_nn_pair(2, m, 2 * m + 5, m) for m in (600, 3000, 4095)],
                      ["last_index", "ties_unordered", "frame0"]),
    "shared_x": (lambda: _nn_shared([0]), ["last_index", "ties_unordered", "frame0"]),
    "shared_xy": (lambda: _nn_shared([0, 1]), ["last_index", "ties_unordered", "frame0"]),
    "signed_zero_x": (_nn_zero_x, ["last_index", "ties_unordered", "frame0"]),
    "far_tiny": (lambda: [tuple(G.far(a) for a in _nn_pair(2, 1024, 2048, 81)),
                          tuple(G.tiny(a) for a in _nn_pair(2, 1024, 2048, 82))], ["last_index", "frame0"]),
    "batch32": (lambda: [_nn_pair(32, 512, 1024, 83)], ["last_index", "ties_unordered", "frame0"]),
    "nonfinite_known": (_nn_nonfinite, ["last_index", "frame0"]),
}


def nn_mutants(names, inputs, refs):
    out = {}
    for nm in names:
        res = []
        for (unk, known), (d2, idx) in zip(inputs, refs):
            if nm == "last_index":
                res.append(G.mut_nn_last_index(idx, d2, known))
            elif nm == "ties_unordered":
                res.append(G.mut_nn_ties_unordered(idx, d2))
            elif nm == "frame0":
                res.append(G.mut_frame0(idx))
        out[nm] = res
    return out


def some_differ(refs, muts):
    """does the mutant differ from the reference on at least one input (refs / muts: parallel lists of arrays or of
    lists of arrays)"""
    for r, m in zip(refs, muts):
        rs, ms = (r, m) if isinstance(r, list) else ([r], [m])
        if any(not np.array_equal(a, b) for a, b in zip(rs, ms)):
            return True
    return False


# ---- inverse-distance weights: d2 [rows,3] ----------------------------------------------------------------------
def weight_inputs(rows, seed):
    rng = np.random.default_rng(seed)
    d2 = np.sort(rng.uniform(0, 0.03, size=(rows, 3)).astype(np.float32) ** 2, axis=1)
    inf = F32(np.inf)
    special = np.array([[0, 1e-4, 4e-4], [0, 0, 1e-4], [0, 0, 0], [1e-4, 1e-4, 1e-4], [1e-4, inf, inf], [0, inf, inf],
                        [1e-4, 4e-4, inf], [inf, inf, inf], [1e-40, 1e-39, 1e-38], [0, 1e-45, 1e-4]], np.float32)
    k = min(rows, len(special) * (rows // 16 // len(special) + 1))
    pos = rng.permutation(rows)[:k]
    d2[pos] = special[np.arange(k) % len(special)]
    return d2
