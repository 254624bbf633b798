"""CPU: the float64 ICP reference (tests/icp_reference.py) pinned to the CPU oracle on every case of tests/test_icp_reference_gpu.py.

The oracle's sums are the reference's float32 products summed in raster order in double, so the two agree to double rounding; the
oracle's step (LU gate, Jacobi pseudo-inverse, Rodrigues, composition) and step64 (numpy's LU and eigh) agree on ok and on T within the
T bar.  The cases themselves are checked to be what they claim: launch shapes, plane normals, branches and spectra."""
import math
from collections import Counter

import numpy as np
import pytest

import icp_cases as ic
import icp_reference as ir

ACC_CASES = [(s, v, p) for s in ic.SIZES for v in ("points", "depth") for p in ic.POSES]
SCENE_CASES = [(s, v) for s in ic.SCENES for v in ic.scene_variants(s)]
_SCENE_STEPS = {}


def test_launch_shape_reproduces_the_table():
    for (cols, rows), want in ic.LAUNCH_TABLE.items():
        assert ir.launch_shape(cols, rows) == want, (cols, rows)
    assert ir.launch_shape(352, 288)[0] == 768 and 352 * 288 == 132 * 768
    assert ir.launch_shape(351, 288)[0] == 256 and ir.launch_shape(1, 1) == (256, 1, 1)


@pytest.mark.parametrize("case", ACC_CASES, ids=ic.acc_id)
def test_sums64_matches_oracle_accumulate(orc, case):
    (cols, rows), variant, pose = case
    curr, prev, Kl, T, dist2, min_cos = ic.accumulate_case(cols, rows, variant, pose)
    r, match, n = ic.oracle_rows(variant, curr, prev, Kl, T, dist2, min_cos)
    fn = orc.icp_accumulate if variant == "points" else orc.icp_accumulate_depth
    want, n_acc = fn(curr[0], curr[1], prev[0], prev[1], Kl, T, float(dist2), float(min_cos))
    s64, abs64, n64 = ir.sums64(r, match)
    assert n == n_acc == n64 == int((match >= 0).sum())
    assert np.all(np.abs(s64 - want) <= 1e-12 * abs64), np.max(np.abs(s64 - want) / np.maximum(abs64, 1e-300))
    assert np.isnan(r[match < 0]).all() and not np.isnan(r[match >= 0]).any()
    assert match.max(initial=-1) < cols * rows
    if cols <= 640:
        assert ir.sensitivity(r, match, ir.sum_bound(ir.launch_shape(cols, rows), abs64)) > 2.0


def test_large_motion_projects_points_from_behind_the_camera_onto_valid_pixels():
    """without the s.z <= 0 test these points would be matched: they are behind the camera, project into the image, land on a valid
    previous point and the case's thresholds are wide open"""
    for cols, rows in ((640, 480), (203, 151)):
        curr, prev, Kl, (R, t), _, _ = ic.accumulate_case(cols, rows, "points", "large")
        P = curr[0][..., :3].reshape(-1, 3).astype(np.float64) @ R.T.astype(np.float64) + t
        fx, fy, cx, cy = Kl
        with np.errstate(all="ignore"):
            u, v = fx * P[:, 0] / P[:, 2] + cx, fy * P[:, 1] / P[:, 2] + cy
        behind = ~np.isnan(P[:, 0]) & (P[:, 2] < 0) & (u >= 0) & (v >= 0) & (u < cols) & (v < rows)
        ui, vi = u[behind].astype(int), v[behind].astype(int)
        assert (~np.isnan(prev[0][vi, ui, 0])).sum() > 100
        out = ~np.isnan(P[:, 0]) & (P[:, 2] > 0) & ~((u >= 0) & (v >= 0) & (u < cols) & (v < rows))
        assert out.sum() > 1000


def _scene_steps(orc, scene, variant):
    """the oracle's estimate loop run step by step: [(level, sums, abs64, inliers, T_in, oracle ok, oracle T)] up to the first failure"""
    key = (scene, variant)
    if key in _SCENE_STEPS:
        return _SCENE_STEPS[key]
    curr, prev = ic.scene_pyramids(scene, variant)
    T = (np.eye(3, dtype=np.float32), np.zeros(3, np.float32))
    out = []
    for lvl, _ in ic.schedule():
        Kl = ic.level_K(ic.K, lvl)
        dist2, min_cos = np.float32(ic.DIST * ic.DIST), np.float32(math.cos(ic.ANGLE))
        r, match, n = ic.oracle_rows(variant, curr[lvl], prev[lvl], Kl, T, dist2, min_cos)
        fn = orc.icp_accumulate if variant == "points" else orc.icp_accumulate_depth
        want, _ = fn(curr[lvl][0], curr[lvl][1], prev[lvl][0], prev[lvl][1], Kl, T, float(dist2), float(min_cos))
        s64, abs64, _ = ir.sums64(r, match)
        assert np.all(np.abs(s64 - want) <= 1e-12 * abs64), (scene, variant, lvl)
        ok, T_new = orc.icp_solve_update(want, T)
        out.append((lvl, want, abs64, n, T, ok, T_new))
        if not ok:
            break
        T = T_new
    _SCENE_STEPS[key] = out
    return out


@pytest.mark.parametrize("scene,variant", SCENE_CASES)
def test_step64_matches_oracle_on_every_scene_step(orc, scene, variant):
    steps = _scene_steps(orc, scene, variant)
    for k, (lvl, sums, _, _, T_in, ok, T) in enumerate(steps):
        st = ir.step64(sums, T_in)
        assert st.ok == ok, (k, lvl, st.branch)
        assert st.within(T), (k, lvl, st.branch, st.error(T))
        assert min(st.margins.values(), default=math.inf) > 1e-9 and st.pivot_margin > 1e3, (k, st.margins, st.pivot_margin)


def test_planes_are_what_they_claim(orc):
    fronto = ic.pyramid_points(ic.plane_depth(640, 480, ic.K), ic.K, 1)[0][1]
    m = ~np.isnan(fronto[..., 0])
    assert m.sum() > 250000 and np.all(fronto[m][:, :2] == 0) and np.all(np.abs(fronto[m][:, 2]) > 0.999)
    tilt1 = ic.pyramid_points(ic.plane_depth(640, 480, ic.K, ic.TILT1), ic.K, 1)[0][1]
    m = ~np.isnan(tilt1[..., 0])
    assert m.sum() > 250000 and np.all(tilt1[m][:, 0] == 0) and (np.abs(tilt1[m][:, 1]) > 0.1).mean() > 0.5
    first = {s: _scene_steps(orc, s, "points")[0] for s in ("plane-fronto", "plane-tilt1", "plane-tilt2", "plane-float")}
    for s in ("plane-fronto", "plane-tilt1"):
        A, _ = ir.unpack(first[s][1])
        assert ir.det_lu(A) == 0 and ir.step64(first[s][1], first[s][4]).branch == "det0/NaN-fail"
    A, _ = ir.unpack(first["plane-tilt2"][1])
    w = np.linalg.eigvalsh(A)
    assert w.min() / w.max() > 1e-4 and ir.step64(first["plane-tilt2"][1], first["plane-tilt2"][4]).branch == "chol"
    # the float-map plane: float rounding makes A indefinite, so the Cholesky rule refuses it while the determinant passes
    A, _ = ir.unpack(first["plane-float"][1])
    w = np.linalg.eigvalsh(A)
    assert w.min() < 0 and abs(w.min()) < 1e-6 * w.max() and not ir.chol_accepts(A)[0] and abs(ir.det_lu(A)) > 1e9 * ir.DET_MIN
    assert ir.step64(first["plane-float"][1], first["plane-float"][4]).branch.startswith("pinv")


@pytest.mark.parametrize("name", [c[0] for c in ic.HOOK_CASES])
def test_step64_matches_oracle_on_hook_systems(orc, name):
    sums, table, T_in = ic.hook_case(name)
    assert np.array_equal(sums, np.asarray(sums, np.float32).astype(np.float64), equal_nan=True), "entries are exact floats"
    fin = np.isfinite(sums)
    assert np.array_equal(ir.fixed_order_sum(table)[fin], sums[fin])
    assert all(math.fsum(table[:, s]) == sums[s] for s in np.flatnonzero(fin))
    if len(table) > 1:
        assert np.all(np.abs(table[:, fin]).max(0) > 0), "every row carries part of every non-zero entry"
    st = ir.step64(sums, T_in)
    ok, T = orc.icp_solve_update(sums, T_in)
    assert st.ok == ok and st.within(T), (st.branch, st.error(T))
    bar = 1e-7 if name in ic.BOUNDARY_CASES else 1e-9
    assert min(st.margins.values(), default=math.inf) > bar and st.pivot_margin > 1e3, (st.margins, st.pivot_margin)


@pytest.mark.parametrize("name", ["tiny-kept", "tiny-dropped"])
def test_the_other_side_of_the_drop_threshold_lies_outside_the_bar(name):
    """A solve that put the tiny direction on the wrong side of 6 DBL_EPSILON wmax (dropped where it must be kept, or inverted where it must
    be dropped) gives a pose the T bar refuses, by far: the hook cases pin the threshold from both sides"""
    sums, _, T_in = ic.hook_case(name)
    st = ir.step64(sums, T_in)
    A, b = ir.unpack(sums)
    r = st.r.copy()
    r[3] = 0.0 if name == "tiny-kept" else b[3] / A[3, 3]
    assert r[3] != st.r[3]
    wrong = st.pose_of(r)
    assert not st.within(wrong) and st.error(wrong) > 1e3, st.error(wrong)
    assert st.kappa < 1e4, "the decoupled tiny direction is solved exactly; the bar follows the condition of the rest"


def test_hook_systems_have_the_spectra_they_claim():
    sy = ic.HOOK_SYSTEMS
    for kap, name in ((1.0, "spd-k1"), (1e3, "spd-k1e3"), (1e6, "spd-k1e6"), (1e8, "spd-k1e8")):
        w = np.linalg.eigvalsh(ir.unpack(ic.pack(*sy[name]))[0])
        assert w.min() > 0 and abs(math.log10(w.max() / w.min() / kap)) < 0.05, (name, w.max() / w.min())
    for name, rel in (("tiny-kept", 1e-14), ("tiny-dropped", 1e-16)):
        A, _ = ir.unpack(ic.pack(*sy[name]))
        w = np.linalg.eigvalsh(A)
        # the tiny eigenvalue is A[3, 3] exactly (its row and column are otherwise zero); eigvalsh finds it only to eps64 wmax
        assert not A[3, :3].any() and not A[3, 4:].any() and abs(A[3, 3] / w.max() / rel - 1) < 1e-6
        assert abs(w.min() / A[3, 3] - 1) < 0.05 and not ir.chol_accepts(A)[0]
        assert abs(ir.det_lu(A)) > 1e12 * ir.DET_MIN
    for name, side in (("sI-above", 1), ("sI-below", -1)):
        s = ir.unpack(ic.pack(*sy[name]))[0][0, 0]
        rel = s ** 6 / 1e-15 - 1
        assert side * rel > 3e-7 and abs(rel) < 2e-6, rel
    assert np.linalg.eigvalsh(ir.unpack(ic.pack(*sy["indefinite"]))[0]).min() < 0


def test_every_branch_is_reached_and_pinv_from_image_data(orc):
    got = Counter()
    for scene, variant in SCENE_CASES:
        for lvl, sums, _, _, T_in, _, _ in _scene_steps(orc, scene, variant):
            b = ir.step64(sums, T_in).branch
            got[b] += 1
            if scene == "plane-float":
                assert b.startswith("pinv"), b
    for name, _, _ in ic.HOOK_CASES:
        sums, _, T_in = ic.hook_case(name)
        got[ir.step64(sums, T_in).branch] += 1
    assert set(got) == set(ir.BRANCHES), got


def test_fixed_order_sum_is_a_sum():
    t = np.random.default_rng(1).standard_normal((131, 27))
    assert np.all(np.abs(ir.fixed_order_sum(t) - t.sum(0)) <= 1e-14 * np.abs(t).sum(0))
