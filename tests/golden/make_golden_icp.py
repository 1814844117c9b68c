"""Golden vectors of my_icp recorded from the REFERENCE ITSELF (build container only).

Imports the unmodified reference lib/utils/icp/icp.py by path (it needs numpy, cv2 and sklearn only)
and records (A, B, init, max_iterations, tolerance) -> (T, distances, i) for the cases below into
icp_cases.npz.  While recording, it asserts that oracle/icp_oracle.py reproduces the reference: the
same i, and T and distances within 1e-12.  The GPU tests read only the npz.

    python tests/golden/make_golden_icp.py          # writes icp_cases.npz + make_golden_icp.log
"""
import importlib.util
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = os.environ.get("PVN3D_REFERENCE", "/root/reference/pvn3d")

from oracle import icp_oracle  # noqa: E402
from pvn3d_b200 import synth  # noqa: E402

BOX = (0.10, 0.06, 0.03)


def load_reference():
    spec = importlib.util.spec_from_file_location("ref_icp", os.path.join(REF, "lib", "utils", "icp", "icp.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def pose(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def cases():
    rng = np.random.default_rng(2026)
    box = synth.box_surface(BOX, 3000, rng)
    big = synth.box_surface((0.16, 0.11, 0.07), 12000, rng)
    R = synth._haar_rotation(rng)
    t = np.array([0.05, -0.03, 0.8])
    out = []

    def scene(ext, R, t, n, faces=None):
        return synth.visible_box_points(ext, R, t, n, 0.001, rng, faces=faces).astype(np.float32)

    B = scene(BOX, R, t, 1300)
    out.append(("visible_5deg_1cm", box, B, pose(*synth.perturb_pose(R, t, 5.0, 0.01, rng)), 500, 1e-9))
    out.append(("visible_15deg_2cm", box, B, pose(*synth.perturb_pose(R, t, 15.0, 0.02, rng)), 500, 1e-9))
    Bo = B.copy()
    k = len(Bo) // 10
    Bo[rng.choice(len(Bo), k, replace=False)] = rng.uniform(B.min(0), B.max(0), size=(k, 3)).astype(np.float32)
    out.append(("outliers_10pct", box, Bo, pose(*synth.perturb_pose(R, t, 5.0, 0.01, rng)), 500, 1e-9))
    # one face only (the 0.10 x 0.06 face, normal +z in the object frame): H is nearly rank 2
    Bf = scene(BOX, R, t, 1300, faces=[4])
    out.append(("flat_face_rank2", box, Bf, pose(*synth.perturb_pose(R, t, 3.0, 0.005, rng)), 500, 1e-9))
    R0, t0 = synth.perturb_pose(np.eye(3), np.zeros(3), 2.0, 0.005, rng)
    B0 = scene(BOX, R0, t0, 1200, faces=[0, 2, 4])
    out.append(("defaults_no_init", box, B0, None, 20, 1e-3))
    out.append(("cap_tol0", box, B, pose(*synth.perturb_pose(R, t, 5.0, 0.01, rng)), 30, 0.0))
    Rb = synth._haar_rotation(rng)
    tb = np.array([-0.1, 0.05, 0.9])
    Bb = scene((0.16, 0.11, 0.07), Rb, tb, 2000)
    out.append(("large_model_12000", big, Bb, pose(*synth.perturb_pose(Rb, tb, 5.0, 0.01, rng)), 500, 1e-9))
    # the reference's icp/test.py shape: 10 random points, B = R(A + t) + noise
    A10 = rng.random((10, 3)).astype(np.float32)
    Rt, _ = synth.perturb_pose(np.eye(3), np.zeros(3), np.rad2deg(0.1 * rng.random()), 0.0, rng)
    B10 = ((A10 + rng.random(3) * 0.1) @ Rt.T + rng.normal(0, 0.01, (10, 3))).astype(np.float32)
    out.append(("ten_points", A10, B10, None, 20, 1e-3))
    return out


def main():
    ref = load_reference()
    log = ["make_golden_icp.py: reference lib/utils/icp/icp.py (my_icp, unmodified)",
           f"numpy {np.__version__}"]
    rec = {}
    names = []
    for k, (name, A, B, init, it, tol) in enumerate(cases()):
        t0 = time.time()
        T, d, i = ref.my_icp(A, B, init, max_iterations=it, tolerance=tol)
        dt = time.time() - t0
        To, do, io = icp_oracle.my_icp(A, B, init, max_iterations=it, tolerance=tol)
        assert io == i, (name, io, i)
        eT, ed = float(np.abs(To - T).max()), float(np.abs(do - d).max())
        assert eT < 1e-12 and ed < 1e-12, (name, eT, ed)
        p = f"c{k}_"
        rec[p + "A"] = A
        rec[p + "B"] = B
        rec[p + "init"] = np.eye(4) if init is None else init
        rec[p + "has_init"] = np.array(init is not None)
        rec[p + "max_iter"] = np.array(it)
        rec[p + "tol"] = np.array(tol)
        rec[p + "T"] = T
        rec[p + "dist"] = d
        rec[p + "i"] = np.array(i)
        names.append(name)
        log.append(f"  case {k} {name}: A {A.shape[0]} pts, B {B.shape[0]} pts, max_iter {it}, tol {tol:g} -> "
                   f"i={i}, mean d={d.mean():.6e} ({dt:.2f}s); oracle: same i, |dT|={eT:.1e}, |dd|={ed:.1e}")
        print(log[-1], flush=True)
    rec["names"] = np.array(names)
    path = os.path.join(HERE, "icp_cases.npz")
    np.savez_compressed(path, **rec)
    log.append(f"wrote {os.path.basename(path)} ({os.path.getsize(path)} bytes): oracle == reference on every case")
    print(log[-1])
    with open(os.path.join(HERE, "make_golden_icp.log"), "w") as f:
        f.write("\n".join(log) + "\n")


if __name__ == "__main__":
    main()
