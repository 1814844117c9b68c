"""Golden vectors of eval_icp's full-resolution scene, recorded from the reference and sklearn (build
container only).

- Back-projection: the reference's own Basic_Utils.dpt_2_cld (lib/utils/basic_utils.py:381-399, the
  method's source taken unmodified from the file; the module itself imports plyfile and the ip_basic
  package, which the recording needs nothing of) on depth images with holes, float32 K and cam_scale.
  Small frames store (cld, choose); the one 480x640 frame stores their SHA-256.
- Label fill: sklearn NearestNeighbors(n_neighbors=1) fitted on a sampled cloud and queried with every
  valid pixel, as fill_label_item (pvn3d/eval_icp.py:388-422) does; `tied` flags the queries whose two
  best float64 squared distances are equal (sklearn may return any of the tied points there).
- End to end, on the 480x640 frame: eval_icp_pvn3d_msk's steps per object (eval_icp.py:224-291) with the
  filled mask -- raster-order pixels of the object, the stride floor(j*cnt/2000) standing in for the
  random subset, skipped below 1500, sklearn MeanShift(bandwidth=0.06, bin_seeding=True) on the float64
  points (labels == 0 kept), then the reference's my_icp(model, cld, init, 500, 1e-9).

While recording, it asserts that oracle/depth_icp_oracle.py agrees: bit-exact back-projection, fill
indices equal on every untied query, and the pipeline's T within 1e-12, same i and kept points.

    python tests/golden/make_golden_depth_icp.py   # writes depth_icp_cases.npz + make_golden_depth_icp.log
"""
import ast
import hashlib
import importlib.util
import os
import sys
import time
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = os.environ.get("PVN3D_REFERENCE", "/root/reference/pvn3d")

from oracle import depth_icp_oracle, icp_oracle  # noqa: E402
from pvn3d_b200 import synth  # noqa: E402

MAX_PTS, MIN_PTS, BW, MAX_ITER, TOL = 2000, 1500, 0.06, 500, 1e-9


def reference_dpt_2_cld():
    """Basic_Utils.dpt_2_cld, unmodified, bound to an object with the reference's xmap / ymap"""
    path = os.path.join(REF, "lib", "utils", "basic_utils.py")
    tree = ast.parse(open(path).read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "Basic_Utils")
    fn = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "dpt_2_cld")
    ns = {"np": np}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), path, "exec"), ns)

    class Utils:  # Basic_Utils.__init__'s maps (basic_utils.py:161-162), for an h x w image
        def __init__(self, h, w):
            self.xmap = np.array([[j for i in range(w)] for j in range(h)])
            self.ymap = np.array([[i for i in range(w)] for j in range(h)])

    return lambda dpt, cam_scale, K: ns["dpt_2_cld"](Utils(*dpt.shape[:2]), dpt, cam_scale, K)


def load_reference_icp():
    spec = importlib.util.spec_from_file_location("ref_icp", os.path.join(REF, "lib", "utils", "icp", "icp.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def sha(*arrays) -> str:
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def brute_nn(cloud, pcld, chunk=256):
    """(index of the first minimum, whether the minimum is tied) per query, float64 brute force"""
    idx = np.empty(len(cloud), np.int64)
    tied = np.empty(len(cloud), bool)
    for s in range(0, len(cloud), chunk):
        d2 = depth_icp_oracle.sqdist64(cloud[s:s + chunk], pcld)
        m = d2.min(1, keepdims=True)
        idx[s:s + chunk] = np.argmin(d2, 1)
        tied[s:s + chunk] = (d2 == m).sum(1) > 1
    return idx, tied


def small_depth(rng, h, w, scale, hole_frac):
    d = np.round(rng.uniform(0.5, 1.5, (h, w)) * scale).astype(np.float32) if scale > 1 else \
        rng.uniform(0.5, 1.5, (h, w)).astype(np.float32)
    d[rng.random((h, w)) < hole_frac] = 0.0
    return d


def backproj_cases(rng):
    k_small = (synth.K_YCB1 * np.array([[0.1], [0.1], [1.0]])).astype(np.float32)     # a 64x48 camera
    k_lm = (synth.K_LINEMOD * np.array([[0.0625], [0.0625], [1.0]])).astype(np.float32)
    edge = np.zeros((16, 16), np.float32)
    f6 = np.float32(1e-6)
    vals = np.array([0.0, f6, np.nextafter(f6, np.float32(1)), np.nextafter(f6, np.float32(0)), -1.0, 1e-7, np.nan,
                     2.5e-6, 65535.0], np.float32)
    edge.ravel()[:] = vals[rng.integers(0, len(vals), 256)]
    return [
        ("holes_ycb_48x64", small_depth(rng, 48, 64, 10000.0, 0.15), np.float32(10000.0), k_small),
        ("metres_linemod_30x40", small_depth(rng, 30, 40, 1.0, 0.1), np.float32(1.0), k_lm),
        ("threshold_values_16x16", edge, np.float32(1000.0), k_small),
    ]


def fill_cases(rng):
    # a 96x128 depth frame with holes, 1500 sampled valid pixels, random labels
    K = (synth.K_YCB1 * np.array([[0.2], [0.2], [1.0]])).astype(np.float32)
    d = small_depth(rng, 96, 128, 10000.0, 0.1)
    cloud, valid = depth_icp_oracle.dpt_2_cld(d, 10000.0, K)
    q = cloud[valid]
    samp = q[np.sort(rng.choice(len(q), 1500, replace=False))]
    out = [("frame_96x128", q, samp, rng.integers(0, 22, 1500).astype(np.int32))]
    # dyadic lattice: queries and points on multiples of 2^-6, duplicated points -> many exact ties
    s6 = 2.0 ** -6
    pts = rng.integers(-8, 8, (400, 3)) * s6
    pts = np.concatenate([pts, pts[:50]])
    qs = rng.integers(-10, 10, (3000, 3)) * s6 + np.where(rng.random((3000, 1)) < 0.3, s6 / 2, 0.0)
    out.append(("dyadic_ties", qs.astype(np.float32), pts.astype(np.float32), rng.integers(0, 22, 450).astype(np.int32)))
    return out


def main():
    import sklearn
    from sklearn.cluster import MeanShift
    from sklearn.neighbors import NearestNeighbors

    ref_d2c = reference_dpt_2_cld()
    ref_icp = load_reference_icp()
    rng = np.random.default_rng(2028)
    log = ["make_golden_depth_icp.py: reference Basic_Utils.dpt_2_cld and my_icp (unmodified), "
           "sklearn NearestNeighbors(n_neighbors=1) and MeanShift(bandwidth=0.06, bin_seeding=True)",
           f"sklearn {sklearn.__version__}, numpy {np.__version__}"]
    rec = {}

    def note(s):
        log.append(s)
        print(s, flush=True)

    # ---- back-projection
    names = []
    for k, (name, dpt, cs, K) in enumerate(backproj_cases(rng)):
        cld, choose = ref_d2c(dpt, cs, K)
        oc, ov = depth_icp_oracle.dpt_2_cld(dpt, cs, K)
        assert cld.dtype == np.float32 and np.array_equal(np.nonzero(ov)[0], choose), name
        assert np.array_equal(oc[ov].view(np.uint32), cld.view(np.uint32)), name
        p = f"bp{k}_"
        rec[p + "dpt"], rec[p + "cam_scale"], rec[p + "K"], rec[p + "cld"], rec[p + "choose"] = dpt, cs, K, cld, choose
        names.append(name)
        note(f"  back-projection {name}: {dpt.shape}, {len(choose)} valid; oracle bit-exact")
    rec["bp_names"] = np.array(names)

    # ---- the 480x640 frame (one frame of the depth batch generator)
    fr = synth.make_icp_depth_batch(1, seed=31)
    dpt, cs, K = fr["depth"][0], fr["cam_scale"][0], fr["K"][0]
    cld, choose = ref_d2c(dpt, cs, K)
    oc, ov = depth_icp_oracle.dpt_2_cld(dpt, cs, K)
    assert np.array_equal(np.nonzero(ov)[0], choose) and np.array_equal(oc[ov].view(np.uint32), cld.view(np.uint32))
    rec["full_dpt"], rec["full_cam_scale"], rec["full_K"] = dpt, cs, K
    rec["full_sha"] = np.array(sha(cld, choose))
    note(f"  back-projection full_frame: {dpt.shape}, {len(choose)} valid; oracle bit-exact; sha256 {rec['full_sha']}")

    # ---- label fill
    names = []
    for k, (name, q, samp, lab) in enumerate(fill_cases(rng)):
        nn = NearestNeighbors(n_neighbors=1).fit(samp)
        ind = nn.kneighbors(q, return_distance=True)[1][:, 0]
        oi, tied = brute_nn(q, samp)
        assert np.array_equal(oi[~tied], ind[~tied]), name
        d2 = depth_icp_oracle.sqdist64(q[tied], samp)
        assert np.all(d2[np.arange(tied.sum()), ind[tied]] == d2.min(1)), name     # sklearn: one of the tied
        p = f"fill{k}_"
        rec[p + "cloud"], rec[p + "pcld"], rec[p + "point_labels"] = q, samp, lab
        rec[p + "index"], rec[p + "labels"], rec[p + "tied"] = ind.astype(np.int32), lab[ind], tied
        names.append(name)
        note(f"  fill {name}: {len(q)} queries, {len(samp)} points, {int(tied.sum())} tied; "
             f"oracle == sklearn on every untied query")
    rec["fill_names"] = np.array(names)

    # fill_label_item on the full frame with the generator's sampled cloud and border-flipped labels
    pcld, plab = fr["pcld"][0], fr["labels"][0]
    t0 = time.time()
    ind = NearestNeighbors(n_neighbors=1).fit(pcld).kneighbors(cld, return_distance=True)[1][:, 0]
    oi, tied = brute_nn(cld, pcld, chunk=128)
    assert np.array_equal(oi[~tied], ind[~tied])
    all_msk = np.zeros(dpt.size, np.uint8)
    all_msk[choose] = plab[ind]
    rec["full_pcld"], rec["full_point_labels"], rec["full_fill"] = pcld, plab, all_msk.reshape(dpt.shape)
    rec["full_fill_tied"] = np.array(int(tied.sum()))
    note(f"  fill full_frame: {len(cld)} queries, {len(pcld)} points, {int(tied.sum())} tied "
         f"({time.time() - t0:.0f}s); oracle == sklearn on every untied query")

    # ---- end to end, eval_item_pvn3d_msk per object
    labels = all_msk.astype(np.int32)                          # 0 on invalid pixels, as the refiner sees it
    full_cloud = oc
    objs = [int(c) for c in np.nonzero(fr["present"][0])[0]]
    done = []
    for c in objs:
        sel = np.nonzero(labels[choose] == c)[0]               # eval_icp indexes the valid-pixel cloud
        if len(sel) < MIN_PTS:
            note(f"  end-to-end class {c}: {len(sel)} pixels < {MIN_PTS}: skipped")
            continue
        if len(sel) > MAX_PTS:
            sel = sel[(np.arange(MAX_PTS) * len(sel)) // MAX_PTS]
        pc = cld[sel]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ms = MeanShift(bandwidth=BW, bin_seeding=True).fit(pc.astype(np.float64))
        kept = np.nonzero(ms.labels_ == 0)[0]
        init = np.identity(4, dtype=np.float32)
        init[:3, :] = fr["init"][0, c]
        model = fr["models"][c]
        T, dist, i = ref_icp.my_icp(model.copy(), pc[kept], init_pose=init, max_iterations=MAX_ITER, tolerance=TOL)
        o = depth_icp_oracle.object_fit(model, full_cloud, labels, c, init.astype(np.float64), MAX_PTS, MIN_PTS, BW,
                                        MAX_ITER, TOL)
        assert o is not None and o[2] == i and np.array_equal(o[3], choose[sel[kept]]), c
        eT = float(np.abs(o[0] - T).max())
        assert eT <= 1e-12, (c, eT)
        p = f"e2e{len(done)}_"
        rec[p + "cls"], rec[p + "T"], rec[p + "i"] = np.array(c), T, np.array(i)
        rec[p + "kept"], rec[p + "err"] = choose[sel[kept]].astype(np.int32), np.array(dist.mean())
        done.append(c)
        note(f"  end-to-end class {c}: {(labels == c).sum()} pixels -> {len(sel)} strided -> {len(kept)} in the "
             f"biggest cluster, my_icp i={i}; oracle: same kept pixels and i, |dT|={eT:.1e}")
        if len(done) == 2:
            break
    assert len(done) == 2
    rec["e2e_n"] = np.array(len(done))
    rec["full_init"], rec["full_present"] = fr["init"][0], fr["present"][0]

    path = os.path.join(HERE, "depth_icp_cases.npz")
    np.savez_compressed(path, **rec)
    note(f"wrote {os.path.basename(path)} ({os.path.getsize(path)} bytes): oracle == reference / sklearn on every case")
    with open(os.path.join(HERE, "make_golden_depth_icp.log"), "w") as f:
        f.write("\n".join(log) + "\n")


if __name__ == "__main__":
    main()
