"""Golden vectors of Basic_Utils.fill_missing recorded from the REFERENCE ITSELF (build container only).

Imports the unmodified reference lib/utils/ip_basic/ip_basic/depth_map_utils_ycb.py by path (numpy and cv2)
and calls fill_in_multiscale exactly as fill_missing does -- on depth / cam_scale * scale_2_80m (float32),
extrapolate False, blur 'bilateral', max_depth 3, show_process True -- then rescales the result by
/ scale_2_80m * cam_scale.  Records the cases below into fill_cases.npz.  While recording it asserts that
tests/depth_fill_ref.py reproduces the reference: the show_process stages s1 .. s6 bit for bit, s7 and the
output within the bilateral bound, and that every wrong reference of depth_fill_ref.MUTANTS is told apart
by at least one case.  Logs the reference's CPU time per 480x640 frame.  The tests read only the npz.

    python tests/golden/make_golden_fill.py          # writes fill_cases.npz + make_golden_fill.log
"""
import importlib.util
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
REF = os.environ.get("PVN3D_REFERENCE", "/root/reference/pvn3d")

import depth_fill_ref as R  # noqa: E402
from depth_fill_cases import CASES, LARGE, OUT_STRIDE, encode_large, load, make_cases  # noqa: E402

if not hasattr(np, "bool"):
    np.bool = bool  # the reference predates numpy 1.24, which removed the np.bool alias


def load_reference():
    path = os.path.join(REF, "lib", "utils", "ip_basic", "ip_basic", "depth_map_utils_ycb.py")
    spec = importlib.util.spec_from_file_location("ref_depth_map_utils_ycb", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def reference_fill(mod, dpt, cam_scale, scale_2_80m):
    """Basic_Utils.fill_missing(dpt, cam_scale, scale_2_80m, show_process=True), one frame"""
    dpt = dpt / cam_scale * scale_2_80m
    final, proc = mod.fill_in_multiscale(dpt.copy(), extrapolate=False, blur_type="bilateral", show_process=True,
                                         max_depth=3.0)
    return final / scale_2_80m * cam_scale, proc


def main():
    mod = load_reference()
    log = []

    def say(s):
        print(s)
        log.append(s)

    out = {}
    rejected = {m: [] for m in R.MUTANTS}
    recorded = {}
    for name, depth, cs, s2s, keep in make_cases():
        rec = {}
        s2s32 = np.float32(s2s)
        for b in range(depth.shape[0]):
            ref_out, proc = reference_fill(mod, depth[b], cs[b], s2s32)
            st = R.fill_stages(depth[b], cs[b], s2s32)
            for k in ("s1", "s2", "s3", "s4", "s5"):
                key = next(x for x in proc if x.startswith(k + "_"))
                assert np.array_equal(st[k], proc[key]), (name, b, k)
            assert np.array_equal(st["s5"], proc["s6_extended_depths"]), (name, b, "s6")
            bound = R.bilateral_bound(st["minmax"])
            e7 = float(np.abs(st["s7"].astype(np.float64) - proc["s7_blurred_depths"]).max())
            eo_px = np.abs(st["out"].astype(np.float64) - ref_out)
            eo = float(eo_px.max())
            assert e7 <= bound, (name, b, e7, bound)
            assert (eo_px <= R.out_bound(st["minmax"], cs[b], s2s32, ref_out)).all(), (name, b, eo)
            for m in R.MUTANTS:
                mst = R.fill_stages(depth[b], cs[b], s2s32, mutant=m)
                if R.mutant_rejected(mst, proc["s4_blurred_depths"], proc["s5_combined_depths"],
                                     proc["s7_blurred_depths"], st["minmax"]):
                    rejected[m].append(f"{name}[{b}]")
            say(f"  {name}[{b}] {depth.shape[1]}x{depth.shape[2]} cam_scale {cs[b]:g} scale_2_80m {s2s:g}: "
                f"valid in {int((depth[b] / cs[b] * s2s32 > R.T).sum())}, s7 {int((proc['s7_blurred_depths'] > R.T).sum())}; "
                f"minmax ({st['minmax'][0]:.4g}, {st['minmax'][1]:.4g}); |s7 - oracle| {e7:.2e} "
                f"(bound {bound:.2e}), |out - oracle| {eo:.2e}")
            for k in keep:
                src = {"s1": proc["s1_inverted_depths"], "s2": proc["s2_dilated_depths"],
                       "s3": proc["s3_closed_depths"], "s4": proc["s4_blurred_depths"],
                       "s5": proc["s5_combined_depths"], "s7": proc["s7_blurred_depths"], "out": ref_out,
                       "out_sub": ref_out[::OUT_STRIDE, ::OUT_STRIDE]}[k]
                rec.setdefault(k, []).append(np.asarray(src, np.float32))
        arrays = {k: np.stack(v) for k, v in rec.items()}
        arrays.update(depth=depth, cam_scale=cs, scale_2_80m=np.float32(s2s))
        if keep == LARGE:
            out.update(encode_large(name, arrays))
        else:
            out.update({f"{name}__{k}": v for k, v in arrays.items()})
        recorded[name] = arrays
    for m, cases in rejected.items():
        say(f"mutant {m}: rejected by {', '.join(cases) if cases else 'NOTHING'}")
        assert cases, m
    # the reference's CPU time per 480x640 frame, on the YCB-shape frames
    ycb = next(c for c in make_cases() if c[0] == "ycb")
    depth, cs = ycb[1], ycb[2]
    times = []
    for rep in range(5):
        for b in range(depth.shape[0]):
            t0 = time.perf_counter()
            reference_fill(mod, depth[b], cs[b], np.float32(1.0))
            times.append(time.perf_counter() - t0)
    import cv2

    say(f"reference fill_missing on the CPU (cv2 {cv2.__version__}, {cv2.getNumThreads()} cv2 threads, "
        f"{os.cpu_count()} cpus): 480x640 frame median {np.median(times) * 1e3:.1f} ms, min {min(times) * 1e3:.1f} ms "
        f"over {len(times)} calls")
    path = os.path.join(HERE, "fill_cases.npz")
    np.savez_compressed(path, case_names=np.array(CASES), **out)
    back = load(path)
    for name, arrays in recorded.items():
        for k, v in arrays.items():
            assert np.array_equal(back[name][k], v), (name, k)   # the encoding is lossless
    say(f"wrote fill_cases.npz ({os.path.getsize(path)} bytes): oracle == reference on every case")
    with open(os.path.join(HERE, "make_golden_fill.log"), "w") as f:
        f.write("\n".join(log) + "\n")


if __name__ == "__main__":
    main()
