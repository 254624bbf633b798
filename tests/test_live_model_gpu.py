"""DF_KINFU_LIVE_MODEL on the GPU: df_mesh_correspond equals its oracle (tests/correspond_oracle.c) bit for bit; the loop's ICP reference maps
and its canonical points are reproduced bit for bit from public entry points (the cloud moved by half a voxel, df_warp, mesh() faces,
df_raster_mesh, df_mesh_correspond); the mode is deterministic, resumes exactly from snapshots, is not disturbed by mesh() / render(), falls
back to the ray-cast loop bit for bit where it must, is switched on by the environment, and holds a static scene still."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from dynamicfusion_b200 import capi, kinfu as kf, synth  # noqa: E402
import color_oracle  # noqa: E402
import correspond_oracle as co  # noqa: E402
import gpu_util as gu  # noqa: E402
import raster_oracle  # noqa: E402
from scenes import K640, look_at, sphere_mesh  # noqa: E402

ROOT = Path(__file__).resolve().parents[1]
FRAMES = [synth.umbrella_depth(t) for t in range(15)]
IDENT = (np.eye(3, dtype=np.float32), np.zeros(3, np.float32))


def _t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a, np.int32 if dtype == torch.int32 else np.float32)).cuda()


def _gpu_correspond(ids, pts, verts, src, tris, w2c, target=None, max_dist=0.0, pad=5):
    """df_mesh_correspond on padded-pitch device maps; returns (points, normals) as numpy"""
    lib = capi.load()
    s = torch.cuda.current_stream().cuda_stream
    rows, cols = ids.shape
    pc = cols + pad
    I = torch.full((rows, pc), -1, dtype=torch.int32, device="cuda"); I[:, :cols] = _t(ids, torch.int32)
    P = torch.full((rows, pc, 4), 3.0, device="cuda"); P[:, :cols] = _t(pts)
    T = None
    if target is not None:
        T = torch.full((rows, pc, 4), 3.0, device="cuda"); T[:, :cols] = _t(target)
    v, sv = _t(verts), _t(src)
    tr = _t(np.asarray(tris, np.int32).reshape(-1, 3), torch.int32)
    op = torch.full((rows, pc, 4), 7.0, device="cuda")
    on = torch.full((rows, pc, 4), 7.0, device="cuda")
    capi.check(lib.df_mesh_correspond(I.data_ptr(), pc * 4, P.data_ptr(), pc * 16, v.data_ptr() if len(v) else None,
                                      sv.data_ptr() if len(sv) else None, len(v), v.shape[1], tr.data_ptr() if len(tr) else None, len(tr),
                                      capi.make_aff(*w2c), cols, rows, T.data_ptr() if T is not None else None, pc * 16, max_dist,
                                      op.data_ptr(), pc * 16, on.data_ptr(), pc * 16, s))
    Op, On = op.cpu().numpy(), on.cpu().numpy()
    assert np.all(Op[:, cols:] == 7.0) and np.all(On[:, cols:] == 7.0)   # nothing written past the image's columns
    return Op[:, :cols], On[:, :cols]


def _same_bits(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def _deformed(cloud, centre):
    d = cloud.copy()
    x = cloud[:, :3].astype(np.float64) - centre
    d[:, :3] = (cloud[:, :3] + 0.01 * np.sin(np.stack([7 * x[:, 1], 5 * x[:, 2], 9 * x[:, 0]], 1))).astype(np.float32)
    return d


# ------------------------------------------------------------------ the kernel ---------------------------------------------------------------
def test_correspond_equals_the_oracle():
    cloud, tris, centre, _, _ = sphere_mesh()
    src = _deformed(cloud, centre)
    rng = np.random.default_rng(3)
    cases = [("front", look_at(centre, 0.8), K640, 640, 480), ("oblique", look_at(centre, 0.5, (0.3, -0.2, 1.0)), K640, 640, 480),
             ("close_up", look_at(centre, 0.24, (-0.1, 0.15, 1.0)), K640, 640, 480),
             ("ragged", look_at(centre, 0.6, (0.2, 0.1, 1.0)), (180.0, 170.0, 61.3, 97.8), 203, 151)]
    for name, w2c, K, cols, rows in cases:
        ids, pts, _, stats = gu.gpu_raster(cloud, tris, w2c, K, cols, rows)
        if name == "close_up":
            assert stats[3] > 0                                          # the large-triangle path drew some of these pixels
        drawn = ids >= 0
        target = pts + rng.uniform(-0.01, 0.01, pts.shape).astype(np.float32)
        target[rng.random(ids.shape) < 0.05] = np.nan
        for source in (cloud, src):
            for tg, md in ((None, 0.0), (target, 0.012)):
                want = co.correspond(ids, pts, cloud, source, tris, w2c, tg, md)
                got = _gpu_correspond(ids, pts, cloud, source, tris, w2c, tg, md)
                assert _same_bits(got[0], want[0]) and _same_bits(got[1], want[1]), (name, tg is None)
                kept = ~np.isnan(want[0][..., 0])
                assert kept.sum() > 1000 and (tg is not None or np.array_equal(kept, drawn)), name
                if tg is not None:
                    assert 0 < (drawn & ~kept).sum() < drawn.sum() // 2          # the distance test removes some pixels, not most
    # xyz rows (vstride 3)
    w2c = look_at(centre, 0.5, (0.3, -0.2, 1.0))
    ids, pts, _, _ = gu.gpu_raster(cloud, tris, w2c, K640, 640, 480)
    want = co.correspond(ids, pts, cloud[:, :3], src[:, :3], tris, w2c)
    got = _gpu_correspond(ids, pts, cloud[:, :3], src[:, :3], tris, w2c)
    assert _same_bits(got[0], want[0]) and _same_bits(got[1], want[1])
    # an empty mesh: no pixel has a triangle
    ids = np.full((48, 64), -1, np.int32)
    pts = np.full((48, 64, 4), np.nan, np.float32)
    got = _gpu_correspond(ids, pts, np.zeros((0, 4), np.float32), np.zeros((0, 4), np.float32), np.zeros((0, 3), np.int32), IDENT)
    assert np.all(np.isnan(got[0])) and np.all(np.isnan(got[1]))


def test_correspond_refuses_bad_pitches_without_writing():
    lib = capi.load()
    s = torch.cuda.current_stream().cuda_stream
    cols, rows = 64, 48
    ids = torch.zeros((rows, cols + 1), dtype=torch.int32, device="cuda")
    pts = torch.zeros((rows, cols + 1, 4), device="cuda")
    v = torch.zeros((3, 4), device="cuda")
    t = torch.tensor([[0, 1, 2]], dtype=torch.int32, device="cuda")
    out = torch.full((rows * (cols + 1) * 4 + 4,), 7.0, device="cuda")
    good = dict(ip=cols * 4, pp=cols * 16, tp=cols * 16, op=cols * 16, np_=cols * 16)
    for bad in (dict(ip=cols * 4 + 2), dict(ip=cols * 4 - 4), dict(pp=cols * 16 + 4), dict(tp=cols * 16 + 8), dict(op=cols * 16 - 16),
                dict(np_=cols * 16 + 4)):
        a = dict(good, **bad)
        st = lib.df_mesh_correspond(ids.data_ptr(), a["ip"], pts.data_ptr(), a["pp"], v.data_ptr(), v.data_ptr(), 3, 4, t.data_ptr(), 1,
                                    capi.make_aff(*IDENT), cols, rows, pts.data_ptr(), a["tp"], 0.1, out.data_ptr(), a["op"], out.data_ptr(),
                                    a["np_"], s)
        assert st != 0, bad
    torch.cuda.synchronize()
    assert torch.all(out == 7.0)


# ------------------------------------------------------------------ the frame loop ------------------------------------------------------------
def _shift(p):
    """R_vol * (vs/2) as the loop forms it: float32, left to right"""
    R = np.array(list(p.volume_pose.R), np.float32).reshape(3, 3)
    h = [np.float32(p.volume_size[d]) / np.float32(p.volume_dims[d]) / np.float32(2) for d in range(3)]
    return np.array([R[r, 0] * h[0] + R[r, 1] * h[1] + R[r, 2] * h[2] for r in range(3)], np.float32)


def _live_mesh(k):
    """(shifted unwarped vertices, shifted warped vertices, faces) of the object's current state, from public entry points"""
    lib = capi.load()
    s = torch.cuda.current_stream().cuda_stream
    cloud, nrm = k.buffer("cloud"), k.buffer("cloud_normals")
    nodes = np.ascontiguousarray(k.buffer("nodes"))
    _, _, faces = k.mesh()
    src = cloud.copy()
    src[:, :3] = src[:, :3] - _shift(k.params)
    P, N, nd = _t(src), _t(nrm), _t(nodes)
    M = len(nodes)
    grid = torch.empty(lib.df_node_grid_bytes(M), dtype=torch.uint8, device="cuda")
    capi.check(lib.df_build_node_grid(nd.data_ptr(), M, grid.data_ptr(), s))
    capi.check(lib.df_warp(nd.data_ptr(), M, grid.data_ptr(), P.data_ptr(), N.data_ptr(), len(src), 4, capi.make_aff(*IDENT), 0, None, None, s))
    return src, P.cpu().numpy(), faces


def _K(p):
    return (p.intr.fx, p.intr.fy, p.intr.cx, p.intr.cy)


def test_icp_reference_is_the_rendered_live_model():
    k = kf.KinFu(gu.kinfu_params(256, kf.LIVE_MODEL, max_nodes=1024, cloud_capacity=1_000_000))
    p = k.params
    ident_w2c = color_oracle.aff_inv(IDENT)                              # dfh_aff_inv of the identity, as the loop forms it
    checked = 0
    for t, d in enumerate(FRAMES[:12]):
        fused = k(d)
        if not fused or k.info()["nodes"] < 8:
            continue
        _, live, faces = _live_mesh(k)
        ids, pts, nrm, _ = gu.gpu_raster(live, faces, ident_w2c, _K(p), p.cols, p.rows)
        assert _same_bits(k.buffer("prev_points"), pts), t
        assert _same_bits(k.buffer("prev_normals"), nrm), t
        assert (ids >= 0).sum() > 50000, t
        checked += 1
    assert checked >= 10 and k.info()["live_model_fallbacks"] == 0
    k.close()


def test_association_is_the_correspondence_on_the_kept_live_mesh():
    k = kf.KinFu(gu.kinfu_params(256, kf.LIVE_MODEL, max_nodes=1024, cloud_capacity=1_000_000))
    p = k.params
    checked = 0
    for t in range(8):
        k(FRAMES[t])
        if t < 2:
            continue
        src, live, faces = _live_mesh(k)
        pose_t = k.getCameraPose()
        nxt = synth.compose(pose_t, (synth.camera_drift(1)[0].astype(np.float32), np.array([0.002, -0.001, 0.0005], np.float32)))
        k.set_overrides(pose=nxt)
        assert k(FRAMES[t + 1])
        cam2model = color_oracle.aff_mul(color_oracle.aff_inv(pose_t), nxt)
        w2c = color_oracle.aff_inv(cam2model)
        ids, pts, _, _ = gu.gpu_raster(live, faces, w2c, _K(p), p.cols, p.rows)
        want = _gpu_correspond(ids, pts, live, src, faces, w2c, k.buffer("curr_points"), p.icp_dist_thres)
        assert _same_bits(k.buffer("canonical_visible"), want[0]), t
        assert (~np.isnan(want[0][..., 0])).sum() > 50000
        oracle = co.correspond(ids, pts, live, src, faces, w2c, k.buffer("curr_points"), p.icp_dist_thres)
        assert _same_bits(oracle[0], want[0]) and _same_bits(oracle[1], want[1])
        checked += 1
    assert checked >= 5
    k.close()


def _state(k):
    return k.state_digest(), k.buffer("prev_points").tobytes(), k.buffer("prev_normals").tobytes()


@pytest.mark.parametrize("extra", [0, kf.WARPED_INTEGRATE | kf.EXTEND_FIELD])
def test_two_objects_agree_after_every_frame(extra):
    a, b = (kf.KinFu(gu.kinfu_params(128, kf.LIVE_MODEL | extra, max_nodes=1024, cloud_capacity=1_000_000)) for _ in range(2))
    for t, d in enumerate(FRAMES):
        assert a(d) == b(d)
        assert _state(a) == _state(b), t
    assert a.info()["live_model_fallbacks"] == 0 and a.info()["resets"] == 0
    a.close()
    b.close()


def test_resume_equals_the_uninterrupted_run(tmp_path):
    ref = kf.KinFu(gu.kinfu_params(128, kf.LIVE_MODEL, max_nodes=1024, cloud_capacity=1_000_000))
    states = []
    snaps = {}
    for t, d in enumerate(FRAMES[:12]):
        ref(d)
        states.append(_state(ref))
        if t in (0, 5):
            snaps[t] = ref.snapshot()
    ref.close()
    for t0, data in snaps.items():
        k = kf.KinFu(gu.kinfu_params(128, kf.LIVE_MODEL, max_nodes=1024, cloud_capacity=1_000_000))
        k.restore(data)
        for t in range(t0 + 1, 12):
            k(FRAMES[t])
            assert _state(k) == states[t], (t0, t)
        k.close()


def test_mesh_and_render_between_frames_change_nothing():
    a, b = (kf.KinFu(gu.kinfu_params(128, kf.LIVE_MODEL, max_nodes=1024, cloud_capacity=1_000_000)) for _ in range(2))
    for t, d in enumerate(FRAMES[:10]):
        a(d)
        b(d)
        b.mesh()
        b.render()
        if b.info()["nodes"] >= 8:
            b.mesh(live=True)
            b.render(live=True)
            b.render((np.eye(3, dtype=np.float32), np.array([0.01, 0.0, 0.0], np.float32)), live=True)
        assert _state(a) == _state(b), t
        assert a.info()["launches"] == b.info()["launches"], t
    a.close()
    b.close()


def _digests(flags, frames, cloud_capacity=1_000_000):
    k = kf.KinFu(gu.kinfu_params(128, flags, max_nodes=1024, cloud_capacity=cloud_capacity))
    out = []
    for d in frames:
        k(d)
        out.append(k.state_digest())
    info = k.info()
    k.close()
    return out, info


def test_fallbacks_equal_the_ray_cast_loop():
    frames = FRAMES[:8]
    base, _ = _digests(0, frames, cloud_capacity=5000)
    live, info = _digests(kf.LIVE_MODEL, frames, cloud_capacity=5000)
    assert live == base
    assert info["live_model_fallbacks"] == len(frames) - 1 and info["cloud_points"] == 5000
    rigid, _ = _digests(kf.RIGID_ONLY, frames)
    rigid_live, info = _digests(kf.RIGID_ONLY | kf.LIVE_MODEL, frames)
    assert rigid_live == rigid and info["live_model_fallbacks"] == 0


def test_environment_switches_it_on():
    code = ("import sys, json; sys.path[:0] = [{root!r}, {tests!r}]\n"
            "import test_live_model_gpu as T\n"
            "from dynamicfusion_b200 import kinfu as kf\n"
            "print(json.dumps(T._digests(0, T.FRAMES[:5])[0]))\n").format(root=str(ROOT), tests=str(ROOT / "tests"))
    env = dict(os.environ, DF_KINFU_LIVE_MODEL="1")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    import json
    got = json.loads(r.stdout.strip().splitlines()[-1])
    want, _ = _digests(kf.LIVE_MODEL, FRAMES[:5])
    off, _ = _digests(0, FRAMES[:5])
    assert got == want and got != off


def test_static_scene_stays_put():
    # The thresholds come from the first run of this test on an H100, not from a model of the error.  That run printed: worst pose 13.594 mm /
    # 0.5159 deg, hit-mask agreement 0.9988, |dz| median 0.3102 voxel, p99 1.1120.  They are set about 1.5 times above it.  The pose drifts
    # on a scene that does not move, which is worth knowing: the translation-only data term has no regulariser, so the warp field can take
    # up a rigid offset as readily as the camera pose can.
    k = kf.KinFu(gu.kinfu_params(256, kf.LIVE_MODEL, max_nodes=1024, cloud_capacity=1_000_000))
    p = k.params
    frames = [synth.umbrella_depth(t, drift=False, shape_t=0) for t in range(10)]
    for d in frames:
        k(d)
    info = k.info()
    assert info["resets"] == 0 and info["frame_counter"] == 10 and info["live_model_fallbacks"] == 0
    worst_t, worst_r = 0.0, 0.0
    for t in range(10):
        R, tr = k.getCameraPose(t)
        worst_t = max(worst_t, float(np.linalg.norm(tr)))
        worst_r = max(worst_r, float(np.degrees(np.arccos(np.clip((np.trace(R.astype(np.float64)) - 1) / 2, -1, 1)))))
    # the ray-cast of the volume at the latest pose (df_raycast_points over the object's own volume)
    lib = capi.load()
    s = torch.cuda.current_stream().cuda_stream
    import ctypes as C
    ptr, pitch, cols, rows = C.c_void_p(), C.c_size_t(), C.c_int(), C.c_int()
    capi.check(lib.df_kinfu_get_buffer(k.h, kf.BUF["volume"], C.byref(ptr), C.byref(pitch), C.byref(cols), C.byref(rows)))
    vs = p.volume_size[0] / p.volume_dims[0]
    V = capi.make_volume(ptr.value, p.volume_dims, [p.volume_size[d] / p.volume_dims[d] for d in range(3)], max(p.tsdf_trunc_dist, 2.1 * vs),
                         p.tsdf_max_weight)
    vol_pose = (np.array(list(p.volume_pose.R), np.float32).reshape(3, 3), np.array(list(p.volume_pose.t), np.float32))
    cam2vol = color_oracle.aff_mul(color_oracle.aff_inv(vol_pose), k.getCameraPose())
    Rinv = color_oracle.aff_inv((cam2vol[0], np.zeros(3, np.float32)))[0]
    rc = torch.empty((p.rows, p.cols, 4), device="cuda")
    rn = torch.empty_like(rc)
    capi.check(lib.df_raycast_points(V, capi.make_aff(*cam2vol), capi.f9(Rinv), p.intr, p.cols, p.rows, p.raycast_step_factor,
                                     p.gradient_delta_factor, rc.data_ptr(), p.cols * 16, rn.data_ptr(), p.cols * 16, s))
    rc, rn = rc.cpu().numpy(), rn.cpu().numpy()
    pts = k.buffer("prev_points")
    k.close()
    hit_r, hit_m = ~np.isnan(rc[..., 2]), ~np.isnan(pts[..., 2])
    uniform = (gu.erode(hit_r) | gu.erode(~hit_r)) & (gu.erode(hit_m) | gu.erode(~hit_m))
    agree = (hit_r == hit_m)[uniform].mean()
    both = gu.erode(hit_r) & gu.erode(hit_m)
    ray = rc[..., :3] / np.linalg.norm(rc[..., :3], axis=-1, keepdims=True)
    cosine = -np.einsum("ijk,ijk->ij", np.nan_to_num(rn[..., :3]), np.nan_to_num(ray))
    sel = both & (cosine > 0.3)
    dz = np.abs(pts[..., 2][sel].astype(np.float64) - rc[..., 2][sel]) / vs
    print(f"static scene: worst pose {worst_t * 1000:.3f} mm / {worst_r:.4f} deg; hit-mask agreement {agree:.4f} over {uniform.sum()} px; "
          f"|dz| over {sel.sum()} px: median {np.median(dz):.4f} voxel, p99 {np.percentile(dz, 99):.4f}, max {dz.max():.3f}")
    assert worst_t <= 0.02 and worst_r <= 0.75
    assert uniform.sum() > 200000 and sel.sum() > 10000
    assert agree >= 0.99
    assert np.median(dz) <= 0.45
    assert np.percentile(dz, 99) <= 1.6
