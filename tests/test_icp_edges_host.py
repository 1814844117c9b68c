"""Without a GPU: the cases of tests/icp_edge_cases.py reach the branches of csrc/icp.cu they are named for (through a
numpy restatement of icp_build_kernel's grid choice), the restated reference equals icp_oracle, and each wrong
reference of icp_edge_cases.MUTANTS differs from the oracle, beyond the tolerance tests/test_icp_edges_gpu.py uses,
on the case it is checked on there -- so a kernel that computed a mutant could not pass the GPU tests."""
import os

import numpy as np
import pytest

import icp_edge_cases as E
from oracle import icp_oracle

ICP_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pvn3d_b200", "csrc", "icp.cu")
TOL_D, TOL_T = 1e-12, 1e-9      # test_icp_edges_gpu.py's step tolerances


def test_restatement_follows_the_kernel_source():
    with open(ICP_CU) as f:
        src = f.read()
    for line in ("constexpr int kMaxCells = 16384;",
                 "const double floor_e = 1e-3 * emax + 1e-9;",
                 "const double target = fmin(static_cast<double>(kMaxCells), 4.0 * np);",
                 "double cell = exp2(rint(log2(cbrt(e[0] * e[1] * e[2] / target))));",
                 "if (prod <= kMaxCells) break;",
                 "h.margin = 1e-6 * cell + 1e-13 * cmax;",
                 "(cell_start[c + 1] > cell_start[c]) ? 0 : 255;",
                 "s_done = fabs(prev - mean) < p.tol;",
                 "const int qpos = static_cast<int>(static_cast<long long>(j) * cnt / nsel);"):
        assert line in src, line


def test_grid_restatement_on_known_models():
    g = E.grid(np.array([[0.0, 0.0, 0.0]], np.float32))
    assert g["dims"].tolist() == [1, 1, 1] and g["target"] == 4.0
    # 2 points 1 m apart on x: e = (1, 1e-3 + 1e-9, 1e-3 + 1e-9), target 8 -> edge 2^-8, 257 cells on x
    g = E.grid(np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0]], np.float32))
    assert g["h"] == 2.0 ** -8 and g["dims"].tolist() == [257, 1, 1] and g["doublings"] == 0
    assert g["dt"].max() == g["dt_true"].max() == 128 and g["counts"].tolist() == [1] + [0] * 255 + [1]


def test_target_cap():
    t = {n: E.grid(E.model(n))["target"] for n in ("pts_4095", "pts_4096", "cap_4097", "pts_16384", "pts_65536")}
    assert t["pts_4095"] == 4 * 4095 < E.MAX_CELLS
    assert t["pts_4096"] == 4 * 4096 == E.MAX_CELLS
    assert t["cap_4097"] == t["pts_16384"] == t["pts_65536"] == E.MAX_CELLS < 4 * 4097


def test_rod_runs_the_doubling_loop():
    A = E.model("rod")
    g = E.grid(A)
    ext = A.max(0).astype(np.float64) - A.min(0)
    assert np.all(ext[1:] < g["floor_e"]) and g["doublings"] >= 1       # the floor sets the thin axes
    first = np.floor((A.max(0) - np.floor(A.min(0) / g["cell0"]) * g["cell0"]) / g["cell0"]) + 1
    assert first.prod() > E.MAX_CELLS and g["dims"].prod() <= E.MAX_CELLS
    for name in ("plane", "line"):                                     # zero-width axes
        Am = E.model(name)
        assert Am[:, 2].min() == Am[:, 2].max() and E.grid(Am)["dims"][2] == 1


def test_gap_is_wider_than_the_capped_transform():
    A = E.model("gap_600")
    g = E.grid(A)
    q = E.queries("gap_600", A, faces=False)["gap"]
    cells = E.cell_index(q, g["lo"], g["h"], g["dims"])
    assert g["dt_true"][cells].min() > E.DT_CAP and np.all(g["dt"][cells] == E.DT_CAP)


def test_outlier_packs_one_cell():
    g = E.grid(E.model("outlier_10m"))
    assert g["counts"].max() >= 500 and g["h"] == 0.25


def test_offset_model_makes_the_float32_centroid_visible():
    A = E.model("offset_50m")
    c32 = A.mean(axis=0).astype(np.float64)                # numpy's float32 mean, as the final fit takes it
    assert np.abs(c32 - A.astype(np.float64).mean(0)).max() > 1e-9
    assert np.abs(E.centre(A) - E.OFFSET).max() < 0.1
    g = E.grid(A)
    assert g["margin"] > 1e-13 * 80                          # the coordinate term of the margin is in play


def test_duplicates_and_faces():
    A = E.model("dups_40")
    uniq, first, counts = np.unique(A, axis=0, return_index=True, return_counts=True)
    assert len(A) - len(uniq) >= 0.3 * len(A)
    g = E.grid(A)
    dup_cells = np.unique(E.cell_index(uniq[counts > 1], g["lo"], g["h"], g["dims"]))
    assert len(dup_cells) > 100                             # spread across cells
    for name in E.NAMES:
        Am = E.model(name)
        gm = E.grid(Am)
        q = E.queries(name, Am, faces=True)["faces"].astype(np.float64)
        k = (q - gm["lo"]) / gm["h"]
        assert np.array_equal(k, np.round(k)), name        # every coordinate of every face query on a face


def test_inits_drive_metric_shrink():
    s = {k: E.metric_shrink(E.init_pose("pts_4096", k)) for k in E.INITS}
    assert s["rigid"] > 1 - 1e-11
    assert 1 - 1e-4 < s["skew_1e-6"] < 1 - 1e-6
    assert abs(s["scale_1.01"] - 0.965) < 1e-3 and abs(s["shear_1e-3"] - 0.9986) < 1e-4


def test_reference_equals_icp_oracle():
    A = E.box_model(seed=3, n=600)
    B, init = E.fit_scene(A, seed=3, n=300)
    for it, tol in ((1, 0.0), (12, 1e-9), (12, 0.0)):
        T0, d0, i0 = icp_oracle.my_icp(A, B, init, it, tol)
        T1, d1, i1 = E.ORACLE.my_icp(A, B, init, it, tol)
        assert i0 == i1 and np.array_equal(T0, T1) and np.array_equal(d0, d1)
    q = np.random.default_rng(0).normal(size=(500, 3)) * 0.05
    pts = np.concatenate([A, A[:100]]).astype(np.float64)
    d0, i0 = icp_oracle.nearest(q, pts)
    d1, i1 = E.brute_nearest(q, pts)
    assert np.array_equal(d0, d1) and np.array_equal(i0, i1)


def test_exact_scene_converges_at_step_zero():
    A, B, init = E.exact_scene()
    means = []
    E.ORACLE.my_icp(A, B, init, 5, 0.0, trace=means)
    assert means[0] == 0.0 and len(means) == 5
    assert E.ORACLE.my_icp(A, B, init, 5, 1e-9)[2] == 0


def test_rank_scenes():
    sc = E.rank_scenes()
    ranks = {}
    for name, (A, B, init) in sc.items():
        src0, idx = E.step_pieces(A, B, init)
        Bd = B.astype(np.float64)
        H = (src0[idx] - src0[idx].mean(0)).T @ (Bd - Bd.mean(0))
        s = np.linalg.svd(H, compute_uv=False)
        ranks[name] = int((s > 1e-12 * max(s[0], 1e-300)).sum())
        assert np.linalg.matrix_rank(np.asarray(A, np.float64) - np.mean(A, 0)) == 3
    assert ranks == {"identical": 0, "collinear": 1, "plane_reflect": 2}
    A, B, init = sc["plane_reflect"]
    src0, idx = E.step_pieces(A, B, init)
    assert E.reflection_det(src0[idx], B.astype(np.float64)) < 0


def test_selection_and_mixed_batches():
    d = E.selection_batch()
    cnt = {c: int((d["mask"][0] == c).sum()) for c in range(E.SEL_N_CLS)}
    assert [cnt[c] for c in range(1, 6)] == [E.SEL_MIN - 1, E.SEL_MIN, E.SEL_MAX, E.SEL_MAX + 1, 2 * E.SEL_MAX + 1]
    assert (d["mask"][1] == E.SEL_WHOLE).all() and d["present"][0, 7] == 1 and cnt[7] == 0
    m = E.mixed_batch()
    assert E.MIX_B * E.MIX_N_CLS > 2048
    from pvn3d_b200.icp import model_table
    _, off = model_table(m["models"], E.MIX_N_CLS)
    sizes = np.diff(off)
    assert len(sizes) == E.MIX_N_CLS and sizes[2] == 1 and sizes[3] == 4097 and sizes[4] == 65536
    assert sizes[1] == sizes[6] == sizes[30] == 0 and sizes[63] == 3000


# ------------------------------------------------------------------------------------------------------------
# each mutant is told apart from the oracle on the case the GPU tests check it on
# ------------------------------------------------------------------------------------------------------------
def _pose_case(name, kind):
    A = E.model(name)
    B = E.apply(E.scene_pose(name), E.all_queries(name, A, faces=False)).astype(np.float32)
    return A, B, E.init_pose(name, kind)


def _step_gap(mutant, A, B, init, it=1, tol=0.0):
    T0, d0, i0 = E.ORACLE.my_icp(A, B, init, it, tol)
    T1, d1, i1 = E.MUTANTS[mutant].my_icp(A, B, init, it, tol)
    return i0 != i1, np.abs(d0 - d1).max(), np.abs(T0 - T1).max()


def test_mutant_tie_highest():
    A = E.model("dups_40")
    q = E.all_queries("dups_40", A, faces=True)
    _, i0 = E.ORACLE.nn(q, A, "cpu")
    _, i1 = E.MUTANTS["tie_highest"].nn(q, A, "cpu")
    assert (i0 != i1).sum() > 100


@pytest.mark.parametrize("mutant,name,kind,what", [("dist_f32", "pts_4096", "rigid", "d"),
                                                   ("model_frame", "pts_4096", "scale_1.01", "d"),
                                                   ("final_f64", "offset_50m", "rigid", "T")])
def test_mutant_pose_channel(mutant, name, kind, what):
    _, dd, dT = _step_gap(mutant, *_pose_case(name, kind))
    assert (dd > TOL_D) if what == "d" else (dT > TOL_T), (dd, dT)


def test_mutant_no_reflection_fix():
    _, _, dT = _step_gap("no_reflection_fix", *E.rank_scenes()["plane_reflect"])
    assert dT > 0.1


def test_mutant_stop_le():
    A, B, init = E.exact_scene()
    di, _, _ = _step_gap("stop_le", A, B, init, it=5, tol=0.0)
    assert di


def test_mutant_select_round():
    d = E.selection_batch()
    gaps = []
    for b, c in ((0, 4), (0, 5), (1, E.SEL_WHOLE)):
        s0 = E.ORACLE.select(d["mask"][b], c, E.SEL_MAX)
        s1 = E.MUTANTS["select_round"].select(d["mask"][b], c, E.SEL_MAX)
        assert len(s0) == len(s1) == E.SEL_MAX and not np.array_equal(s0, s1)
        init = np.eye(4)
        init[:3] = d["init"][b, c].astype(np.float64)
        T0 = E.ORACLE.my_icp(d["models"][c], d["pcld"][b][s0], init, 3, 1e-9)[0]
        T1 = E.ORACLE.my_icp(d["models"][c], d["pcld"][b][s1], init, 3, 1e-9)[0]
        gaps.append(np.abs(T0 - T1).max())
    assert min(gaps) > TOL_T, gaps
    for c, cnt in ((2, E.SEL_MIN), (3, E.SEL_MAX)):          # at or below max_pts the two rules agree
        assert np.array_equal(E.ORACLE.select(d["mask"][0], c, E.SEL_MAX),
                              E.MUTANTS["select_round"].select(d["mask"][0], c, E.SEL_MAX))


def test_every_mutant_has_a_host_check():
    checked = {"tie_highest", "dist_f32", "model_frame", "final_f64", "no_reflection_fix", "stop_le", "select_round"}
    assert set(E.MUTANTS) == checked
