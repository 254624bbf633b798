"""Projective ICP on the GPU against the float64 reference (tests/icp_reference.py), kernel by kernel and iteration by iteration.

Accumulate: every image size of icp_cases.LAUNCH_TABLE, both variants, three poses, through the C ABI with dense and with padded pitches.
The launch shape is pinned by which partial rows get written, the 27 sums are held entry by entry to the bar of sum_bound (float per-thread
sums and float warp trees), and the bar is small enough that one dropped or doubled correspondence exceeds it.  Estimate: the VGA pyramid
is run once per prefix of its 19-step schedule, and each step's partials and pose are checked against the reference at the pose the GPU
read.  Solve tail: df_icp_solve_step on systems of chosen spectrum.  Every branch class of the reference's prediction of the device rule
is reached, with every decision it rests on guarded by a margin.  The file runs once more with programmatic dependent launch off."""
import ctypes as C
import math
import os
import subprocess
import sys
from collections import Counter

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("orc")]

import icp_cases as ic  # noqa: E402
import icp_reference as ir  # noqa: E402
from dynamicfusion_b200 import capi  # noqa: E402
import gpu_util as gu  # noqa: E402

SCRATCH = 32 + 27 * 1024                                   # DF_ICP_SCRATCH_DOUBLES
SENTINEL = -1.2345e300
PADS4 = (3, 1, 5, 2)                                       # float4 elements of padding per row: vcurr, ncurr, vprev, nprev
PADS2 = (1, 3)                                             # u16 elements of padding per row: dcurr, dprev
ACC_CASES = [(s, v, p) for s in ic.SIZES for v in ("points", "depth") for p in ic.POSES]
SCENE_CASES = [(s, v) for s in ic.SCENES for v in ic.scene_variants(s)]
_EST, _HOOK = {}, {}
IDENTITY = (np.eye(3, dtype=np.float32), np.zeros(3, np.float32))


def _dev(a, pad=0):
    """(device tensor, pitch in bytes) of a (rows, cols, 4) float32 or (rows, cols) uint16 map, each row followed by `pad` elements of
    NaN / 0xFFFF"""
    rows, cols = a.shape[:2]
    if a.dtype == np.uint16:
        buf = np.full((rows, cols + pad), 0xFFFF, np.uint16)
        buf[:, :cols] = a
        return torch.from_numpy(buf.view(np.int16)).cuda(), (cols + pad) * 2
    buf = np.full((rows, cols + pad, 4), np.nan, np.float32)
    buf[:, :cols] = a
    return torch.from_numpy(buf).cuda(), (cols + pad) * 16


def _scratch():
    return torch.full((SCRATCH,), SENTINEL, dtype=torch.float64, device="cuda")


def _accumulate(variant, curr, prev, Kl, T, dist2, min_cos, padded=False):
    """scratch after df_icp_accumulate(_depth), as float64 numpy"""
    pads = (PADS2[0], PADS4[1], PADS2[1], PADS4[3]) if variant == "depth" else PADS4
    maps = [_dev(m, p if padded else 0) for m, p in zip((curr[0], curr[1], prev[0], prev[1]), pads)]
    scratch = _scratch()
    rows, cols = curr[1].shape[:2]
    lib = capi.load()
    fn = lib.df_icp_accumulate if variant == "points" else lib.df_icp_accumulate_depth
    args = [x for t, p in maps for x in (t.data_ptr(), p)]
    capi.check(fn(*args, cols, rows, capi.make_intr(*Kl), capi.make_aff(*T), float(dist2), float(min_cos), scratch.data_ptr(), gu.stream()))
    torch.cuda.synchronize()
    return scratch.cpu().numpy()


def _check_table(scratch, blocks, finite=True):
    """the launch shape: partial rows < blocks written (finite for finite inputs), every row from `blocks` on, and scratch[27:32],
    still holding the sentinel; returns the written table"""
    table = scratch[32:].reshape(1024, 27)
    assert np.all(table[blocks:] == SENTINEL), "partial rows past the launch's block count were written"
    assert np.all(scratch[27:32] == SENTINEL)
    assert not np.any(table[:blocks] == SENTINEL), "a block did not write its partial row"
    if finite:
        assert np.all(np.isfinite(table[:blocks]))
    return table[:blocks]


@pytest.mark.parametrize("case", ACC_CASES, ids=ic.acc_id)
def test_accumulate_matches_float64_reference(case):
    (cols, rows), variant, pose = case
    curr, prev, Kl, T, dist2, min_cos = ic.accumulate_case(cols, rows, variant, pose)
    r, match, n = ic.oracle_rows(variant, curr, prev, Kl, T, dist2, min_cos)
    s64, abs64, _ = ir.sums64(r, match)
    shape = ir.launch_shape(cols, rows)
    bar = ir.sum_bound(shape, abs64)

    scratch = _accumulate(variant, curr, prev, Kl, T, dist2, min_cos)
    table = _check_table(scratch, shape[1])
    S = scratch[:27]
    assert np.all(np.abs(S - table.sum(0)) <= 1e-15 * np.abs(table).sum(0))
    assert np.array_equal(S, ir.fixed_order_sum(table)), "the reduction's fixed order"
    err = np.abs(S - s64)
    assert np.all(err <= bar), (np.max(err / np.maximum(bar, 1e-300)), int(np.argmax(err / np.maximum(bar, 1e-300))))
    ratio = float(np.max(np.where(bar > 0, err / np.maximum(bar, 1e-300), 0.0)))
    print(f"\n[icp accumulate] {cols}x{rows} {variant} {pose}: inliers {n}, launch {shape}, max |S - S64| / bar = {ratio:.3g}")
    if cols <= 640:
        assert ir.sensitivity(r, match, bar) > 2.0, "one correspondence more or less could hide under the bar"

    # padded pitches with NaN / 0xFFFF in the padding: the pixel-to-thread mapping ignores the pitch, so the result is the same bits
    padded = _accumulate(variant, curr, prev, Kl, T, dist2, min_cos, padded=True)
    assert np.array_equal(padded.view(np.uint64), scratch.view(np.uint64))


@pytest.mark.parametrize("variant", ["points", "depth"])
def test_nan_normals_follow_the_reference_rule(variant):
    """a NaN current normal at a valid point passes the cosine test (NaN comparisons are false) and the row is formed as usual; a NaN
    previous normal at a matched point passes too, and its NaN row makes every sum NaN and the step fail"""
    cols, rows = 320, 240
    curr, prev, Kl, T, dist2, min_cos = ic.accumulate_case(cols, rows, variant, "offset")
    _, match, n0 = ic.oracle_rows(variant, curr, prev, Kl, T, dist2, min_cos)
    inl = np.flatnonzero(match.reshape(-1) >= 0)
    nc = curr[1].copy()
    nc.reshape(-1, 4)[inl[::97], :3] = np.nan
    curr_n = (curr[0], nc)
    r, match, n = ic.oracle_rows(variant, curr_n, prev, Kl, T, dist2, min_cos)
    assert n >= n0 and np.all(match.reshape(-1)[inl[::97]] >= 0)
    s64, abs64, _ = ir.sums64(r, match)
    shape = ir.launch_shape(cols, rows)
    scratch = _accumulate(variant, curr_n, prev, Kl, T, dist2, min_cos)
    _check_table(scratch, shape[1])
    assert np.all(np.abs(scratch[:27] - s64) <= ir.sum_bound(shape, abs64))

    _, match, _ = ic.oracle_rows(variant, curr, prev, Kl, T, dist2, min_cos)
    npv = prev[1].copy()
    npv.reshape(-1, 4)[match.reshape(-1)[inl[::50]], :3] = np.nan
    prev_n = (prev[0], npv)
    r, match, _ = ic.oracle_rows(variant, curr, prev_n, Kl, T, dist2, min_cos)
    s64, _, _ = ir.sums64(r, match)
    assert np.isnan(s64).all()
    scratch = _accumulate(variant, curr, prev_n, Kl, T, dist2, min_cos)
    _check_table(scratch, shape[1], finite=False)
    assert np.isnan(scratch[:27]).all()
    T_out, ok, _ = _estimate(variant, [curr], [prev_n], [1], levels=1, K0=Kl)
    assert ok == 0 and np.array_equal(T_out[0], IDENTITY[0]) and np.array_equal(T_out[1], IDENTITY[1])


# ------------------------------------------------------------------ estimate, step by step -------------------------------------------------
def _estimate(variant, curr, prev, iters, levels=3, padded=False, K0=ic.K, scratch=None):
    """df_icp_estimate(_depth) from the identity with per-level iteration counts: (T as (R, t), ok, scratch)"""
    lib = capi.load()
    L = levels
    pads = [(2 * l + 1) if padded else 0 for l in range(L)]
    keep = []

    def ptrs(maps, i):
        out = []
        for lvl in range(L):
            t, p = _dev(maps[lvl][i], pads[lvl])
            keep.append(t)
            out.append((t.data_ptr(), p))
        return out

    vc, ncur, vp, npr = ptrs(curr, 0), ptrs(curr, 1), ptrs(prev, 0), ptrs(prev, 1)
    arr = lambda xs: (C.c_void_p * L)(*[x[0] for x in xs])
    cols = (C.c_int * L)(*[curr[l][1].shape[1] for l in range(L)])
    rows = (C.c_int * L)(*[curr[l][1].shape[0] for l in range(L)])
    it = (C.c_int * L)(*iters[:L])
    Tdev = torch.zeros(12, dtype=torch.float32, device="cuda")
    okdev = torch.zeros(1, dtype=torch.int32, device="cuda")
    scratch = _scratch() if scratch is None else scratch
    if variant == "points":
        assert all(a[1] == b[1] == c[1] == d[1] for a, b, c, d in zip(vc, ncur, vp, npr))
        pitch = (C.c_size_t * L)(*[x[1] for x in vc])
        capi.check(lib.df_icp_estimate(arr(vc), arr(ncur), arr(vp), arr(npr), cols, rows, pitch, L, it, capi.make_intr(*K0), ic.DIST,
                                       ic.ANGLE, Tdev.data_ptr(), okdev.data_ptr(), scratch.data_ptr(), gu.stream()))
    else:
        dpitch = (C.c_size_t * L)(*[x[1] for x in vc])
        npitch = (C.c_size_t * L)(*[x[1] for x in ncur])
        capi.check(lib.df_icp_estimate_depth(arr(vc), arr(ncur), arr(vp), arr(npr), cols, rows, dpitch, npitch, L, it, capi.make_intr(*K0),
                                             ic.DIST, ic.ANGLE, Tdev.data_ptr(), okdev.data_ptr(), scratch.data_ptr(), gu.stream()))
    torch.cuda.synchronize()
    T = Tdev.cpu().numpy()
    return (T[:9].reshape(3, 3).copy(), T[9:].copy()), int(okdev.item()), scratch.cpu().numpy()


def _estimate_run(scene, variant):
    """per step k = 1..19: dict(level, branch, sum error / bar, T error / bar); asserts every check of the step on the way"""
    key = (scene, variant)
    if key in _EST:
        return _EST[key]
    curr, prev = ic.scene_pyramids(scene, variant)
    sched = ic.schedule()
    T_prev, ok_prev = IDENTITY, 1
    T0, ok0, _ = _estimate(variant, curr, prev, ic.prefix_iters(0))
    assert ok0 == 1 and np.array_equal(T0[0], IDENTITY[0]) and np.array_equal(T0[1], IDENTITY[1])
    dist2, min_cos = np.float32(ic.DIST * ic.DIST), np.float32(math.cos(ic.ANGLE))
    recs = []
    for k in range(1, len(sched) + 1):
        lvl = sched[k - 1][0]
        T_k, ok_k, scratch = _estimate(variant, curr, prev, ic.prefix_iters(k))
        shape = ir.launch_shape(*curr[lvl][1].shape[1::-1])
        table = _check_table(scratch, shape[1], finite=False)
        where = (scene, variant, k, lvl)
        if not ok_prev:                                    # after a failure: nothing moves, the passes sum nothing
            assert ok_k == 0 and np.all(table == 0), where
            assert np.array_equal(T_k[0], T_prev[0]) and np.array_equal(T_k[1], T_prev[1]), where
            recs.append(dict(level=lvl, branch="-", sum_ratio=0.0, T_ratio=0.0))
            continue
        r, match, _ = ic.oracle_rows(variant, curr[lvl], prev[lvl], ic.level_K(ic.K, lvl), T_prev, dist2, min_cos)
        s64, abs64, _ = ir.sums64(r, match)
        S = ir.fixed_order_sum(table)
        bar = ir.sum_bound(shape, abs64)
        assert np.all(np.isfinite(table)) == np.all(np.isfinite(s64)), where
        err = np.abs(S - s64)
        fin = np.isfinite(s64)
        assert np.all(err[fin] <= bar[fin]) and np.array_equal(np.isnan(S), np.isnan(s64)), (where, np.max(err[fin] / bar[fin]))
        st = ir.step64(S, T_prev)
        assert ok_k == int(st.ok), (where, st.branch, st.det)
        assert st.within(T_k), (where, st.branch, st.error(T_k))
        assert min(st.margins.values(), default=math.inf) > 1e-9 and st.pivot_margin > 1e3, (where, st.margins, st.pivot_margin)
        recs.append(dict(level=lvl, branch=st.branch, sum_ratio=float(np.max(np.where(bar[fin] > 0, err[fin] / np.maximum(bar[fin], 1e-300), 0),
                                                                         initial=0.0)), T_ratio=st.error(T_k)))
        T_prev, ok_prev = T_k, ok_k

    # the whole schedule on padded per-level pitches (NaN / 0xFFFF padding): the dense run's pose, bit for bit
    T_pad, ok_pad, _ = _estimate(variant, curr, prev, ic.ITERS, padded=True)
    assert ok_pad == ok_prev and np.array_equal(T_pad[0].view(np.uint32), T_prev[0].view(np.uint32))
    assert np.array_equal(T_pad[1].view(np.uint32), T_prev[1].view(np.uint32))
    _EST[key] = (recs, T_prev, ok_prev)
    return _EST[key]


@pytest.mark.parametrize("scene,variant", SCENE_CASES)
def test_estimate_step_by_step(scene, variant):
    recs, T, ok = _estimate_run(scene, variant)
    counts = Counter(r["branch"] for r in recs)
    print(f"\n[icp estimate] {scene} {variant}: ok {ok}, branches {dict(counts)}, max sum error / bar "
          f"{max(r['sum_ratio'] for r in recs):.3g}, max T error / bar {max(r['T_ratio'] for r in recs):.3g}")
    if scene in ("umbrella", "sphere-wall", "plane-tilt2"):
        assert ok == 1 and counts["chol"] == len(recs)
    if scene in ("plane-fronto", "plane-tilt1"):
        assert ok == 0 and recs[0]["branch"] == "det0/NaN-fail"
    if scene == "nan-prev":                                # the first finest-level step has nothing to match against
        first0 = next(i for i, r in enumerate(recs) if r["level"] == 0)
        assert ok == 0 and recs[first0]["branch"] == "det0/NaN-fail"
    if scene == "plane-float":
        assert ok == 1 and all(r["branch"].startswith("pinv") for r in recs)


# ------------------------------------------------------------------ solve tail -------------------------------------------------------------
def _hook_run(name, ok_in=1, offset=0):
    sums, table, T_in = ic.hook_case(name)
    n = len(table)
    buf = torch.full((27 * n + 2,), np.nan, dtype=torch.float64, device="cuda")   # the slack double after an odd table holds NaN
    buf[offset:offset + 27 * n] = torch.from_numpy(table.reshape(-1)).cuda()
    Tdev = torch.from_numpy(np.concatenate([T_in[0].reshape(9), T_in[1]]).astype(np.float32)).cuda()
    okdev = torch.full((1,), ok_in, dtype=torch.int32, device="cuda")
    status = capi.load().df_icp_solve_step(buf.data_ptr() + 8 * offset, n, Tdev.data_ptr(), okdev.data_ptr(), gu.stream())
    torch.cuda.synchronize()
    T = Tdev.cpu().numpy()
    return status, (T[:9].reshape(3, 3).copy(), T[9:].copy()), int(okdev.item()), sums, T_in


@pytest.mark.parametrize("name", [c[0] for c in ic.HOOK_CASES])
def test_solve_tail_matches_float64_reference(name):
    status, T, ok, sums, T_in = _hook_run(name)
    capi.check(status)
    st = ir.step64(sums, T_in)
    assert ok == int(st.ok), (st.branch, st.det)
    assert st.within(T), (st.branch, st.error(T))
    if not st.ok:
        assert np.array_equal(T[0], T_in[0]) and np.array_equal(T[1], T_in[1])
    # no decision lies within 1e-9 of its threshold, except the deliberate ones, which lie 1e-6 away with exact float entries; no Cholesky
    # pivot lies within a thousand rounding errors of its threshold
    margin = min(st.margins.values(), default=math.inf)
    assert margin > (1e-7 if name in ic.BOUNDARY_CASES else 1e-9) and st.pivot_margin > 1e3, (st.margins, st.pivot_margin)
    _HOOK[name] = st.branch
    print(f"\n[icp solve tail] {name}: {st.branch}, ok {ok}, kappa_eff {st.kappa:.3g}, T error / bar {st.error(T):.3g}")


def test_solve_tail_skips_after_failure_and_checks_alignment():
    status, T, ok, _, T_in = _hook_run("spd-k1e3", ok_in=0)
    capi.check(status)
    assert ok == 0 and np.array_equal(T[0], T_in[0]) and np.array_equal(T[1], T_in[1])
    status, _, _, _, _ = _hook_run("spd-k1e3", offset=1)
    assert status != 0, "a table that is not 16-byte aligned is refused"


def test_every_branch_is_reached():
    """Every branch class of step64 occurs.  The class is the reference's prediction of the device rule (the device reports only ok and T);
    every step checked guards the decisions it rests on (pivot, determinant and eigenvalue margins), so the device cannot decide otherwise
    without its T or ok leaving the reference's."""
    got = Counter()
    for scene, variant in SCENE_CASES:
        recs = _estimate_run(scene, variant)[0]
        got.update(r["branch"] for r in recs if r["branch"] != "-")
        if scene == "plane-float":                          # from image data, not only through the hook
            assert any(r["branch"].startswith("pinv") for r in recs)
    for name, _, _ in ic.HOOK_CASES:
        if name not in _HOOK:
            test_solve_tail_matches_float64_reference(name)
        got[_HOOK[name]] += 1
    assert set(got) == set(ir.BRANCHES), got


# ------------------------------------------------------------------ programmatic dependent launch off -------------------------------------
def umbrella_T_hex():
    """the umbrella's full estimate (points variant), as hex of the 12 floats"""
    curr, prev = ic.scene_pyramids("umbrella", "points")
    T, ok, _ = _estimate("points", curr, prev, ic.ITERS)
    return f"{ok}:" + np.concatenate([T[0].reshape(9), T[1]]).astype(np.float32).tobytes().hex()


def test_pdl_off_in_subprocess():
    """DF_PDL is read once per process: the whole file again with it off, and one estimate's pose compared bit for bit across the modes"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, DF_PDL="0")
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_icp_reference_gpu.py", "-q", "-m", "gpu", "-k", "not subprocess"],
                       cwd=root, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and "failed" not in r.stdout
    code = "import sys; sys.path[:0] = ['tests', '.']; import test_icp_reference_gpu as t; print(t.umbrella_T_hex())"
    r = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.strip().splitlines()[-1] == umbrella_T_hex()
