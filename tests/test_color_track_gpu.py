"""Colour tracking on the GPU: df_frame_intensity and df_model_intensity equal tests/color_track_oracle.c bit for bit, df_icp_accumulate_color
stays within the float64 bar and equals df_icp_accumulate at weight 0, df_icp_estimate_color follows the float64 steps, the frame loop can be
rebuilt from the public entries, leaves depth-only frames alone, resumes from snapshots, refuses what it must -- and tracks the textured
wall that geometry alone cannot."""
import ctypes as C
import math
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("orc")]

import color_camera_oracle as cco  # noqa: E402
import color_oracle as co  # noqa: E402
import color_track_oracle as cto  # noqa: E402
import color_track_reference as ctr  # noqa: E402
import icp_cases as ic  # noqa: E402
import icp_reference as ir  # noqa: E402
from dynamicfusion_b200 import build, capi, kinfu as kf, synth  # noqa: E402
import gpu_util as gu  # noqa: E402

ROOT = Path(__file__).resolve().parents[1]
SCRATCH = 32 + 27 * 1024
W, MAXR = capi.COLOR_TRACK_WEIGHT, capi.COLOR_TRACK_MAX_RESIDUAL
KV2 = ((1620.0, 1620.0, 959.5, 539.5), 1920, 1080)                   # a Kinect-v2-like colour camera, 52 mm beside the depth camera
D2C = (np.eye(3, dtype=np.float32), np.array([-0.052, 0.0, 0.0], np.float32))


def _pad(a, extra, fill):
    """(device tensor of a with `extra` more elements per row, pitch in bytes)"""
    rows, cols = a.shape[:2]
    host = np.full((rows, cols + extra) + a.shape[2:], fill, a.dtype)
    host[:, :cols] = a
    view = {np.dtype(np.uint32): np.int32, np.dtype(np.uint16): np.int16}.get(host.dtype)
    return torch.from_numpy(host.view(view) if view else host).cuda(), host.strides[0]


def _arr(ctype, xs):
    return (ctype * len(xs))(*xs)


# ------------------------------------------------------------------------------------------------------------ the intensity kernels
def _gpu_frame_intensity(bgra, levels, cols, rows, cam=None, K=None, points=None, cmap=None, trunc=0.0, pad=0):
    img, bp = _pad(bgra, pad, 7)
    sizes = cto.level_sizes(cols, rows, levels)
    outs = [_pad(np.zeros((r, c), np.float32), pad, 0) for c, r in sizes]
    args = [None, 0, None, 0]
    if cam is not None:
        pts, pp = _pad(points, pad, np.nan)
        m, mp = _pad(cmap, pad, 0)
        args = [pts.data_ptr(), pp, m.data_ptr(), mp]
    camst = capi.make_color_camera(cam.K, cam.cols, cam.rows, cam.d2c) if cam is not None else None
    capi.check(capi.load().df_frame_intensity(img.data_ptr(), bp, None if camst is None else C.byref(camst), capi.make_intr(*(K or (1, 1, 0, 0))),
                                              args[0], args[1], args[2], args[3], float(trunc), levels,
                                              _arr(C.c_int, [c for c, _ in sizes]), _arr(C.c_int, [r for _, r in sizes]),
                                              _arr(C.c_void_p, [o.data_ptr() for o, _ in outs]), _arr(C.c_size_t, [p for _, p in outs]), gu.stream()))
    torch.cuda.synchronize()
    return [o.cpu().numpy()[:, :c] for (o, _), (c, r) in zip(outs, sizes)]


@pytest.mark.parametrize("cols,rows,pad", [(640, 480, 0), (203, 151, 5)])
def test_frame_intensity_registered(cols, rows, pad):
    rng = np.random.default_rng(cols)
    bgra = rng.integers(0, 256, (rows, cols, 4), dtype=np.uint8)
    got = _gpu_frame_intensity(bgra, 4, cols, rows, pad=pad)
    want = cto.frame_intensity(bgra, 4)
    assert all(gu.same_bits(g, w) for g, w in zip(got, want))


def test_frame_intensity_through_the_colour_camera():
    K = synth.DEFAULT_K
    cam = cco.Camera(KV2[1], KV2[2], KV2[0], D2C)
    depth, bgra = synth.umbrella_rgbd(0, color_camera=(KV2[0], KV2[1], KV2[2], D2C))
    from oracle import orc
    pts = orc.points_normals(K, orc.bilateral(depth, 7, 4.5, 0.04))[0]
    cmap = cco.depth_map(depth, K, cam)
    got = _gpu_frame_intensity(bgra, 3, 640, 480, cam=cam, K=K, points=pts, cmap=cmap, trunc=0.04, pad=3)
    want = cto.frame_intensity(bgra, 3, camera=cam, K_depth=K, points=pts, color_map=cmap, trunc_dist=0.04)
    assert all(gu.same_bits(g, w) for g, w in zip(got, want))
    no_occl = cto.frame_intensity(bgra, 1, camera=cam, K_depth=K, points=pts, color_map=np.full_like(cmap, 0x7f000000), trunc_dist=0.04)[0]
    occluded = np.isnan(want[0]) & ~np.isnan(no_occl) & ~np.isnan(pts[..., 0])
    assert occluded.sum() > 50                                      # the small sphere hides part of the wall from the colour camera
    assert (~np.isnan(want[0])).mean() > 0.7                        # borders, dropouts and occlusion leave the rest


def _volume_from_poses(frames, poses, K, dim=128):
    from oracle import orc
    dims, vs = (dim,) * 3, (1.0 / dim,) * 3
    vol_pose = synth.volume_pose(1.0)
    colors = np.zeros(dim ** 3, np.uint32)
    for (d, c), P in zip(frames, poses):
        P = tuple(np.asarray(x, np.float32) for x in P)
        co.integrate_color(colors, dims, vs, 0.04, 64, orc.compute_dists(d, K), c, co.aff_mul(co.aff_inv(P), vol_pose), K)
    return colors, dims, vs, vol_pose


def _gpu_model(colors, dims, vs, cam2vol, pyr, pad=0):
    V = capi.make_volume(None, dims, vs, 0.04, 64)
    cols_ = torch.from_numpy(colors.view(np.int32)).cuda()
    pts = [_pad(p, pad, np.nan) for p in pyr]
    outs = [_pad(np.zeros(p.shape, np.float32), pad, 0) for p in pyr]
    L = len(pyr)
    capi.check(capi.load().df_model_intensity(V, cols_.data_ptr(), capi.make_aff(*cam2vol), L, _arr(C.c_int, [p.shape[1] for p in pyr]),
                                              _arr(C.c_int, [p.shape[0] for p in pyr]), _arr(C.c_void_p, [t.data_ptr() for t, _ in pts]),
                                              _arr(C.c_size_t, [q for _, q in pts]), _arr(C.c_void_p, [t.data_ptr() for t, _ in outs]),
                                              _arr(C.c_size_t, [q for _, q in outs]), gu.stream()))
    torch.cuda.synchronize()
    return [t.cpu().numpy()[:, :p.shape[1]] for (t, _), p in zip(outs, pyr)]


@pytest.mark.parametrize("scene", ["c2", "wall"])
def test_model_intensity_equals_the_oracle(scene):
    K = synth.DEFAULT_K
    if scene == "c2":
        frames, poses = [synth.umbrella_rgbd(t) for t in (0, 4, 8)], [synth.camera_drift(t) for t in (0, 4, 8)]
    else:
        frames, poses = [synth.textured_wall_rgbd(t) for t in (0, 4, 8)], [synth.wall_drift(t) for t in (0, 4, 8)]
    colors, dims, vs, vol_pose = _volume_from_poses(frames, poses, K)
    for (d, _), P in zip(frames, poses):
        pyr = [v for v, _ in ic.pyramid_points(d, K, 3)]
        cam2vol = co.aff_mul(co.aff_inv(vol_pose), tuple(np.asarray(x, np.float32) for x in P))
        got = _gpu_model(colors, dims, vs, cam2vol, pyr, pad=2)
        want = [cto.model_intensity(colors, dims, vs, cam2vol, p) for p in pyr]
        assert all(gu.same_bits(g, w) for g, w in zip(got, want))
        assert (~np.isnan(want[0][..., 0])).mean() > 0.3


# ------------------------------------------------------------------------------------------------------------ the ICP kernels
def _gpu_accumulate_color(curr, prev, icurr, model, K, T, dist2, min_cos, weight, pad=0):
    maps = [_pad(m, pad, np.nan) for m in (curr[0], curr[1], prev[0], prev[1], icurr, model)]
    scratch = torch.full((SCRATCH,), -1.2345e300, dtype=torch.float64, device="cuda")
    rows, cols = icurr.shape
    args = [x for t, p in maps for x in (t.data_ptr(), p)]
    capi.check(capi.load().df_icp_accumulate_color(*args, cols, rows, capi.make_intr(*K), capi.make_aff(*T), float(dist2), float(min_cos),
                                                   float(weight), float(MAXR), scratch.data_ptr(), gu.stream()))
    torch.cuda.synchronize()
    return scratch.cpu().numpy()


def _gpu_accumulate(curr, prev, K, T, dist2, min_cos):
    maps = [_pad(m, 0, np.nan) for m in (curr[0], curr[1], prev[0], prev[1])]
    scratch = torch.full((SCRATCH,), -1.2345e300, dtype=torch.float64, device="cuda")
    rows, cols = curr[0].shape[:2]
    args = [x for t, p in maps for x in (t.data_ptr(), p)]
    capi.check(capi.load().df_icp_accumulate(*args, cols, rows, capi.make_intr(*K), capi.make_aff(*T), float(dist2), float(min_cos),
                                             scratch.data_ptr(), gu.stream()))
    torch.cuda.synchronize()
    return scratch.cpu().numpy()


@pytest.fixture(scope="module")
def wall():
    return ctr.wall_pair(0, 1)


@pytest.fixture(scope="module")
def c2():
    return ctr.c2_pair(0, 1)


@pytest.mark.parametrize("level", [0, 1])                         # 640 x 480: 768-thread blocks; 320 x 240: 256-thread blocks
@pytest.mark.parametrize("scene", ["wall", "c2"])
def test_accumulate_color_within_the_float64_bar(scene, level, request):
    P = request.getfixturevalue(scene)
    Kl = ic.level_K(P["K"], level)
    dist2, min_cos = ctr.thresholds()
    T = (np.eye(3, dtype=np.float32), np.array([0.0015, -0.0005, 0.0], np.float32))
    curr, prev, icurr, model = P["curr"][level], P["prev"][level], P["icurr"][level], P["model"][level]
    geo, match, pho = ctr.level_rows(curr, prev, icurr, model, Kl, T, dist2, min_cos)
    S64, A64, n1, n2 = ctr.sums64(geo, match, pho)
    assert n2 > 0.3 * n1
    rows, cols = icurr.shape
    shape = ctr.launch_shape(cols, rows)
    dense = _gpu_accumulate_color(curr, prev, icurr, model, Kl, T, dist2, min_cos, W)
    bar = ir.sum_bound(shape, A64)
    err = np.abs(dense[:27] - S64)
    assert np.all(err <= bar), (err / bar).max()
    print(f"{scene} level {level}: rows {n1} + {n2}, max |S - S64| / bar {float((err / bar).max()):.3f}")
    padded = _gpu_accumulate_color(curr, prev, icurr, model, Kl, T, dist2, min_cos, W, pad=3)
    assert np.array_equal(dense[:27], padded[:27])
    zero = _gpu_accumulate_color(curr, prev, icurr, model, Kl, T, dist2, min_cos, 0.0)
    assert np.array_equal(zero[:27], _gpu_accumulate(curr, prev, Kl, T, dist2, min_cos)[:27])


def _gpu_estimate_color(P, iters, pad=0):
    curr, prev, icurr, model = P["curr"], P["prev"], P["icurr"], P["model"]
    L = len(curr)
    keep = []

    def dev(m):
        t, p = _pad(m, pad, np.nan)
        keep.append(t)
        return t.data_ptr(), p
    vc = [dev(c[0]) for c in curr]; nc = [dev(c[1]) for c in curr]
    vp = [dev(p[0]) for p in prev]; np_ = [dev(p[1]) for p in prev]
    ii = [dev(i) for i in icurr]; mm = [dev(m) for m in model]
    T = torch.zeros(16, dtype=torch.float32, device="cuda")
    ok = torch.zeros(4, dtype=torch.int32, device="cuda")
    scratch = torch.zeros(SCRATCH, dtype=torch.float64, device="cuda")
    ptrs = lambda xs: _arr(C.c_void_p, [a for a, _ in xs])
    capi.check(capi.load().df_icp_estimate_color(ptrs(vc), ptrs(nc), ptrs(vp), ptrs(np_), ptrs(ii), _arr(C.c_size_t, [p for _, p in ii]),
                                                 ptrs(mm), _arr(C.c_size_t, [p for _, p in mm]), _arr(C.c_int, [c[0].shape[1] for c in curr]),
                                                 _arr(C.c_int, [c[0].shape[0] for c in curr]), _arr(C.c_size_t, [p for _, p in vc]), L,
                                                 _arr(C.c_int, list(iters)), capi.make_intr(*P["K"]), float(ctr.DIST), float(ctr.ANGLE),
                                                 float(W), float(MAXR), T.data_ptr(), ok.data_ptr(), scratch.data_ptr(), gu.stream()))
    torch.cuda.synchronize()
    t = T.cpu().numpy()
    return bool(ok.cpu().numpy()[0]), (t[:9].reshape(3, 3).copy(), t[9:12].copy()), scratch.cpu().numpy()


@pytest.mark.parametrize("scene", ["wall", "c2"])
def test_estimate_color_every_step_against_step64(scene, request):
    P = request.getfixturevalue(scene)
    dist2, min_cos = ctr.thresholds()
    T_prev = ctr.IDENTITY
    worst = 0.0
    for k, (lvl, _) in enumerate(ic.schedule(), 1):
        ok, T, scratch = _gpu_estimate_color(P, ic.prefix_iters(k))
        Kl = ic.level_K(P["K"], lvl)
        geo, match, pho = ctr.level_rows(P["curr"][lvl], P["prev"][lvl], P["icurr"][lvl], P["model"][lvl], Kl, T_prev, dist2, min_cos)
        S64, A64, _, _ = ctr.sums64(geo, match, pho)
        # the step's own partial sums (the last accumulate's table), in the solve's fixed order, within the bar of the float64 sums; then the
        # pose against the float64 step from those sums (an ill-conditioned system would magnify the sums' float rounding otherwise)
        rows, cols = P["icurr"][lvl].shape
        shape = ctr.launch_shape(cols, rows)
        S = ir.fixed_order_sum(scratch[32:32 + 27 * shape[1]].reshape(shape[1], 27))
        assert np.all(np.abs(S - S64) <= ir.sum_bound(shape, A64)), k
        st = ir.step64(S, T_prev)
        assert ok == st.ok
        assert st.within(T), (k, st.error(T))
        worst = max(worst, st.error(T))
        T_prev = T
    ok, T, _ = _gpu_estimate_color(P, ic.ITERS, pad=2)               # padded pitches: the same pose
    assert np.array_equal(T[0], T_prev[0]) and np.array_equal(T[1], T_prev[1])
    e, ang = ctr.pose_error(T, P["truth"])
    print(f"{scene}: worst step error / bar {worst:.3f}; pair error {e * 1000} mm, {ang:.4f} deg")


# ------------------------------------------------------------------------------------------------------------ the frame loop
WALL = [synth.textured_wall_rgbd(t) for t in range(21)]


@pytest.mark.parametrize("overlap", ["1", "0"])
def test_loop_rebuilt_from_the_public_entries(monkeypatch, overlap):
    monkeypatch.setenv("DF_KINFU_OVERLAP_EXTRACT", overlap)
    k = kf.KinFu(gu.kinfu_params(128, kf.COLOR | kf.COLOR_TRACKING, max_nodes=1024, cloud_capacity=1_000_000))
    p = k.params
    K = (p.intr.fx, p.intr.fy, p.intr.cx, p.intr.cy)
    vs = (1.0 / 128,) * 3
    vol_pose = synth.volume_pose(1.0)
    k(*WALL[0])
    for t in range(1, 5):
        prev = [(k.buffer("prev_points", l), k.buffer("prev_normals", l)) for l in range(3)]
        colors = k.buffer("color_volume").copy()
        pose_prev = k.getCameraPose()
        assert k(*WALL[t])
        curr = [(k.buffer("curr_points", l), k.buffer("curr_normals", l)) for l in range(3)]
        icurr = [k.buffer("intensity", l) for l in range(3)]
        model = [k.buffer("model_intensity", l) for l in range(3)]
        assert all(gu.same_bits(a, b) for a, b in zip(icurr, cto.frame_intensity(WALL[t][1], 3)))
        cam2vol = co.aff_mul(co.aff_inv(vol_pose), pose_prev)
        assert all(gu.same_bits(m, cto.model_intensity(colors, (128,) * 3, vs, cam2vol, pv[0])) for m, pv in zip(model, prev))
        ok, T, _ = _gpu_estimate_color(dict(curr=curr, prev=prev, icurr=icurr, model=model, K=K), list(p.icp_iter_num)[:3])
        assert ok
        pose = co.aff_mul(pose_prev, T)
        got = k.getCameraPose()
        assert np.array_equal(got[0], pose[0]) and np.array_equal(got[1], pose[1])
    k.close()


def test_depth_only_frames_and_launch_counts():
    a, b = (kf.KinFu(gu.kinfu_params(128, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000)),
            kf.KinFu(gu.kinfu_params(128, kf.COLOR | kf.COLOR_TRACKING, max_nodes=1024, cloud_capacity=1_000_000)))
    for t in range(4):                                                # depth-only frames: the same state, the same launches
        a(WALL[t][0]); b(WALL[t][0])
        assert gu.state(a) == gu.state(b) and a.info()["launches"] == b.info()["launches"]
    a.close(); b.close()
    # colour frames of C2, which geometry tracks too (so both runs take the same branches): the pyramid (3 levels) and, after the first
    # frame, the model maps
    a, b = (kf.KinFu(gu.kinfu_params(128, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000)),
            kf.KinFu(gu.kinfu_params(128, kf.COLOR | kf.COLOR_TRACKING, max_nodes=1024, cloud_capacity=1_000_000)))
    for t in range(4):
        d, c = synth.umbrella_rgbd(t)
        a(d, c); b(d, c)
        assert a.info()["resets"] == b.info()["resets"] == 0
        assert b.info()["launches"] - a.info()["launches"] == (3 if t == 0 else 4)
    d = synth.umbrella_depth(4)
    a(d); b(d)
    assert b.info()["launches"] == a.info()["launches"]
    a.close(); b.close()


def _run_sequence(frames, truth, flags, dim=256, cam=None):
    k = kf.KinFu(gu.kinfu_params(dim, flags, max_nodes=1024, cloud_capacity=1_000_000))
    if cam is not None:
        k.set_color_camera(*cam)
    errs = []
    for t, (d, c) in enumerate(frames):
        k(d, c)
        R, tr = k.getCameraPose()
        Rt, tt = truth(t)
        errs.append((float(tr[0] - tt[0]), math.degrees(math.atan2(R[1, 0], R[0, 0])) - math.degrees(math.atan2(Rt[1, 0], Rt[0, 0])),
                     float(np.linalg.norm(tr - tt))))
    info = k.info()
    k.close()
    return info["resets"], errs


@pytest.mark.parametrize("rigid", [True, False], ids=["rigid_only", "default"])
def test_the_textured_wall_is_tracked_with_colour_only(rigid):
    extra = kf.RIGID_ONLY if rigid else 0
    resets, errs = _run_sequence(WALL, synth.wall_drift, kf.COLOR | extra)
    print(f"geometry: resets {resets}, x error at frame 20 {errs[-1][0] * 1000:.2f} mm")
    assert resets > 0 or abs(errs[-1][0]) > 0.020
    resets, errs = _run_sequence(WALL, synth.wall_drift, kf.COLOR | kf.COLOR_TRACKING | extra)
    print("colour: x error mm", [round(e[0] * 1000, 2) for e in errs], "roll error deg", [round(e[1], 3) for e in errs])
    assert resets == 0
    assert all(abs(e[0]) < 0.004 and abs(e[1]) < 0.3 for e in errs)


def test_the_textured_wall_through_the_colour_camera():
    cam_t = (KV2[0], KV2[1], KV2[2], D2C)
    frames = [(WALL[t][0], synth.textured_wall_rgbd(t, color_camera=cam_t)[1]) for t in range(21)]
    resets, errs = _run_sequence(frames, synth.wall_drift, kf.COLOR | kf.COLOR_TRACKING, cam=(KV2[0], KV2[1], KV2[2], D2C))
    print("colour camera: x error mm", [round(e[0] * 1000, 2) for e in errs], "roll error deg", [round(e[1], 3) for e in errs])
    assert resets == 0
    assert all(abs(e[0]) < 0.004 and abs(e[1]) < 0.3 for e in errs)


def test_c2_rgbd_is_tracked():
    frames = [synth.umbrella_rgbd(t) for t in range(30)]
    resets, errs = _run_sequence(frames, synth.camera_drift, kf.COLOR | kf.COLOR_TRACKING)
    r0, e0 = _run_sequence(frames, synth.camera_drift, kf.COLOR)
    print(f"C2 30 frames: colour tracking |t| error at 30 {errs[-1][2] * 1000:.2f} mm (max {max(e[2] for e in errs) * 1000:.2f}); "
          f"default loop {e0[-1][2] * 1000:.2f} mm (max {max(e[2] for e in e0) * 1000:.2f})")
    assert resets == 0


def test_snapshot_resume_equals_the_uninterrupted_run():
    frames = WALL[:10]
    k = kf.KinFu(gu.kinfu_params(128, kf.COLOR | kf.COLOR_TRACKING, max_nodes=1024, cloud_capacity=1_000_000))
    states = []
    snap = None
    for t, f in enumerate(frames):
        k(*f)
        states.append(gu.state(k))
        if t == 4:
            snap = k.snapshot()
    k.close()
    r = kf.KinFu(gu.kinfu_params(128, kf.COLOR | kf.COLOR_TRACKING, max_nodes=1024, cloud_capacity=1_000_000))
    r.restore(snap)
    for t in range(5, 10):
        r(*frames[t])
        assert gu.state(r) == states[t]
    r.close()


def test_refusals_and_the_environment(capfd, monkeypatch):
    for flags, word in ((kf.COLOR_TRACKING, "DF_KINFU_COLOR"), (kf.COLOR | kf.COLOR_TRACKING | kf.USE_DEPTH, "DF_KINFU_USE_DEPTH"),
                        (kf.COLOR | kf.COLOR_TRACKING | kf.LIVE_MODEL, "DF_KINFU_LIVE_MODEL")):
        with pytest.raises(RuntimeError):
            kf.KinFu(gu.kinfu_params(128, flags, max_nodes=1024, cloud_capacity=1_000_000))
        assert word in capfd.readouterr().err
    monkeypatch.setenv("DF_KINFU_COLOR_TRACKING", "1")
    k, plain = (kf.KinFu(gu.kinfu_params(128, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000)),
                kf.KinFu(gu.kinfu_params(128, 0, max_nodes=1024, cloud_capacity=1_000_000)))
    k(*WALL[0]); plain(WALL[0][0])
    assert k.buffer("intensity").shape == (480, 640)                    # the flag is on
    with pytest.raises(RuntimeError):
        plain.buffer("intensity")                                       # a colourless object is left as it was
    k.close(); plain.close()


def test_cpp_mirror_gives_the_python_poses(tmp_path):
    exe = build.build_cpp_program(ROOT / "tests" / "cpp" / "color_export.cpp", ROOT / "tests" / "cpp" / "_build" / "color_export")
    frames = WALL[:5]
    np.stack([d for d, _ in frames]).tofile(tmp_path / "depth.u16")
    np.stack([c for _, c in frames]).tofile(tmp_path / "bgra.u8")
    env = dict(os.environ, DF_KINFU_COLOR_TRACKING="1")
    r = subprocess.run([str(exe), str(tmp_path / "depth.u16"), str(tmp_path / "bgra.u8"), str(len(frames)), str(tmp_path / "cpp.ply"),
                        str(tmp_path / "cpp.bgra")], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stdout + r.stderr
    p = kf.KinFuParams.default_params_dynamicfusion()
    p.flags = kf.COLOR | kf.COLOR_TRACKING
    k = kf.KinFu(p)
    for depth, bgra in frames:
        k(depth, bgra)
    k.save_mesh(tmp_path / "py.ply", live=True, colors=True)           # the mesh is in the live frame: its vertices carry the poses
    k.close()
    assert (tmp_path / "cpp.ply").read_bytes() == (tmp_path / "py.ply").read_bytes()
