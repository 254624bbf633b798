"""The rasteriser on the GPU (df_raster_mesh, df_kinfu_render): maps, triangle indices and stats equal the oracle's (tests/raster_oracle.c)
bit for bit on an analytic sphere from several poses (one close enough to use the large-triangle path), a 256^3 canonical mesh, a live mesh,
a ragged image and an empty mesh; the frame loop's render equals the oracle on its own mesh, changes no state, writes nothing when it
fails, agrees with the loop's ray-cast, shades like renderImage, and is exported identically by the C++ mirror."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from dynamicfusion_b200 import capi, kinfu as kf, synth  # noqa: E402
import color_oracle as co  # noqa: E402
import gpu_util as gu  # noqa: E402
import mesh_oracle  # noqa: E402
import raster_oracle  # noqa: E402
from oracle import orc  # noqa: E402
from scenes import IDENT, K640, look_at, sphere_mesh  # noqa: E402

ROOT = Path(__file__).resolve().parents[1]
FRAMES = [synth.umbrella_depth(t) for t in range(10)]


def _same(got, want):
    gi, gp, gn, gs = got
    wi, wp, wn, ws = want
    if gi is not None:
        assert np.array_equal(gi, wi)
    assert np.array_equal(gp.view(np.uint32), wp.view(np.uint32))
    assert np.array_equal(gn.view(np.uint32), wn.view(np.uint32))
    if gs is not None:
        assert np.array_equal(gs, ws), (gs, ws)


def _check(verts, tris, w2c, K, cols, rows):
    want = raster_oracle.raster(verts, tris, w2c, K, cols, rows)
    _same(gu.gpu_raster(verts, tris, w2c, K, cols, rows), want)
    return want


def test_sphere_from_three_poses_equals_the_oracle():
    cloud, tris, centre, _, _ = sphere_mesh()
    for name, w2c in (("front", look_at(centre, 0.8)), ("oblique", look_at(centre, 0.5, (0.3, -0.2, 1.0))),
                      ("close_up", look_at(centre, 0.24, (-0.1, 0.15, 1.0)))):
        ids, _, _, stats = _check(cloud, tris, w2c, K640, 640, 480)
        assert stats[4] > 10000, name
        if name == "close_up":
            assert stats[3] > 0                                          # the large-triangle path is exercised
    # xyz rows (vstride 3) and no index map give the same maps
    w2c = look_at(centre, 0.5, (0.3, -0.2, 1.0))
    want = raster_oracle.raster(cloud, tris, w2c, K640, 640, 480)
    got = gu.gpu_raster(np.ascontiguousarray(cloud[:, :3]), tris, w2c, K640, 640, 480, with_ids=False)
    _same(got, (None,) + want[1:])


def test_canonical_mesh_of_c1_256_equals_the_oracle():
    vol, dims, vs, trunc = gu.c1_volume()
    cloud = orc.extract_cloud(vol, dims, (vs,) * 3, trunc, 64, IDENT, 3 * int(np.prod(dims)))
    tris = mesh_oracle.mesh(vol, dims, len(cloud))
    assert tris is not None and len(tris) > 100000
    p = kf.KinFuParams.default_params_dynamicfusion()
    K = (p.intr.fx, p.intr.fy, p.intr.cx, p.intr.cy)
    vol2cam = (np.eye(3, dtype=np.float32), np.array([-0.5, -0.5, 0.5], np.float32))     # the volume pose of KinFuParams.set_volume
    _, _, _, stats = _check(cloud, tris, vol2cam, K, 640, 480)
    assert stats[4] > 50000


def test_live_mesh_after_six_frames_equals_the_oracle():
    k = gu.run(gu.kinfu_params(128, 0, max_nodes=1024, cloud_capacity=1_000_000), FRAMES[:6])
    assert k.info()["nodes"] >= 8
    v, _, f = k.mesh(live=True)
    R, t = k.getCameraPose()
    k.close()
    _, _, _, stats = _check(v, f, co.aff_inv((R, t)), K640, 640, 480)
    assert stats[4] > 1000


def test_ragged_image_with_off_centre_intrinsics():
    cloud, tris, centre, _, _ = sphere_mesh()
    _check(cloud, tris, look_at(centre, 0.6, (0.2, 0.1, 1.0)), (180.0, 170.0, 61.3, 97.8), 203, 151)


def test_empty_mesh_draws_nothing():
    verts = np.zeros((5, 4), np.float32)
    ids, pts, nrm, stats = gu.gpu_raster(verts, np.zeros((0, 3), np.int32), IDENT, K640, 64, 48)
    assert np.all(ids == -1) and np.all(np.isnan(pts)) and np.all(np.isnan(nrm)) and np.all(stats == 0)
    ids, pts, nrm, stats = gu.gpu_raster(np.zeros((0, 4), np.float32), np.zeros((0, 3), np.int32), IDENT, K640, 64, 48)
    assert np.all(ids == -1) and np.all(np.isnan(pts)) and np.all(stats == 0)


def test_skips_and_bad_indices_are_counted_on_the_gpu():
    cloud, tris, centre, _, _ = sphere_mesh()
    bad = tris.copy()
    bad[::7, 1] = len(cloud) + 5                                         # out of range
    bad[3::11, 2] = -2
    near = cloud.copy()
    near[::13, 2] = centre[2] - 0.8 + 0.005                       # a few vertices in front of the near plane
    w2c = look_at(centre, 0.8)
    for verts, tri in ((cloud, bad), (near, tris)):
        _, _, _, stats = _check(verts, tri, w2c, K640, 640, 480)
        assert stats[1] > 0


# ------------------------------------------------------------------ the frame loop ------------------------------------------------------------
def _render_dev(k, live):
    p = k.params
    pts = torch.full((p.rows, p.cols, 4), 7.0, dtype=torch.float32, device="cuda")
    nrm = torch.full((p.rows, p.cols, 4), 7.0, dtype=torch.float32, device="cuda")
    ids = torch.full((p.rows, p.cols), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    st = k.lib.df_kinfu_render(k.h, int(live), None, ids.data_ptr(), p.cols * 4, pts.data_ptr(), p.cols * 16, nrm.data_ptr(), p.cols * 16)
    return st, ids.cpu().numpy(), pts.cpu().numpy(), nrm.cpu().numpy()


def test_kinfu_render_equals_the_oracle_on_its_mesh():
    k = gu.run(gu.kinfu_params(128, 0, max_nodes=1024, cloud_capacity=1_000_000), FRAMES[:6])
    p = k.params
    K = (p.intr.fx, p.intr.fy, p.intr.cx, p.intr.cy)
    R, t = k.getCameraPose()
    moved = (R, t + np.array([0.02, -0.01, -0.05], np.float32))
    for live in (False, True):
        v, _, f = k.mesh(live)
        defaults = (None, (np.eye(3, dtype=np.float32), np.zeros(3, np.float32)) if live else (R, t))
        for pose, cam2model in (defaults, (moved, moved)):
            pts, nrm, ids = k.render(pose, live)
            want = raster_oracle.raster(v, f, co.aff_inv(cam2model), K, p.cols, p.rows)
            _same((ids, pts, nrm, None), want)
            assert (ids >= 0).sum() > 1000
    k.close()


@pytest.mark.parametrize("overlap", ["1", "0"])
def test_rendering_every_frame_changes_nothing(monkeypatch, overlap):
    monkeypatch.setenv("DF_KINFU_OVERLAP_EXTRACT", overlap)
    a, b = (kf.KinFu(gu.kinfu_params(128, 0, max_nodes=1024, cloud_capacity=1_000_000)) for _ in range(2))
    for t, d in enumerate(FRAMES[:8]):
        a(d)
        b(d)
        b.render()
        if b.info()["nodes"] >= 8:
            b.render(live=True)
        assert a.state_digest() == b.state_digest(), t
        assert a.info()["launches"] == b.info()["launches"], t
    a.close()
    b.close()


def test_failures_write_nothing():
    k = gu.run(gu.kinfu_params(128, kf.RIGID_ONLY, max_nodes=1024, cloud_capacity=1_000_000), FRAMES[:3])
    assert k.info()["nodes"] < 8
    st, ids, pts, nrm = _render_dev(k, 1)
    assert st != 0 and np.all(ids == -7) and np.all(pts == 7.0) and np.all(nrm == 7.0)
    with pytest.raises(RuntimeError):
        k.render(live=True)
    k.close()
    k = gu.run(gu.kinfu_params(128, 0, max_nodes=1024, cloud_capacity=2000), FRAMES[:4])  # the cloud is cut at 2000 points
    assert k.info()["cloud_points"] == 2000
    before = k.state_digest()
    st, ids, pts, nrm = _render_dev(k, 0)
    assert st != 0 and np.all(ids == -7) and np.all(pts == 7.0) and np.all(nrm == 7.0)
    assert k.state_digest() == before
    k.close()


def test_canonical_render_agrees_with_the_loops_raycast():
    k = gu.run(gu.kinfu_params(128, 0, max_nodes=1024, cloud_capacity=1_000_000), FRAMES)
    p = k.params
    vs = p.volume_size[0] / p.volume_dims[0]
    R, t = k.getCameraPose()
    Rvol = np.array(list(p.volume_pose.R), np.float32).reshape(3, 3)
    # extraction places voxel i at (i + 1/2) vs, the ray-cast at i vs: move the camera by the same half voxel
    shifted = (R, (t + Rvol @ np.full(3, vs / 2, np.float32)).astype(np.float32))
    pts, _, ids = k.render(shifted)
    rc, rn = k.buffer("prev_points"), k.buffer("prev_normals")
    k.close()
    hit_r, hit_m = ~np.isnan(rc[..., 2]), ids >= 0
    # hit masks at least 2 px from either map's silhouette: pixels whose 5 x 5 neighbourhood is all hit or all miss in each map (so a
    # disagreement there is a region, not an edge pixel)
    uniform = (gu.erode(hit_r) | gu.erode(~hit_r)) & (gu.erode(hit_m) | gu.erode(~hit_m))
    agree = (hit_r == hit_m)[uniform].mean()
    both = gu.erode(hit_r) & gu.erode(hit_m)
    ray = rc[..., :3] / np.linalg.norm(rc[..., :3], axis=-1, keepdims=True)
    cosine = -np.einsum("ijk,ijk->ij", np.nan_to_num(rn[..., :3]), np.nan_to_num(ray))
    sel = both & (cosine > 0.3)
    dz = np.abs(pts[..., 2][sel].astype(np.float64) - rc[..., 2][sel]) / vs
    print(f"hit-mask agreement {agree:.4f} over {uniform.sum()} px; |dz| over {sel.sum()} px: median {np.median(dz):.4f} voxel, "
          f"p99 {np.percentile(dz, 99):.4f}, max {dz.max():.3f}")
    assert uniform.sum() > 200000 and sel.sum() > 10000
    assert agree >= 0.99
    assert np.median(dz) <= 0.25
    assert np.percentile(dz, 99) <= 1.0


def test_render_image_shades_the_render_maps():
    k = gu.run(gu.kinfu_params(128, 0, max_nodes=1024, cloud_capacity=1_000_000), FRAMES[:6])
    p = k.params
    lib = capi.load()
    s = torch.cuda.current_stream().cuda_stream
    light = (C.c_float * 3)(*p.light_pose)
    for live in (False, True):
        pts, nrm, _ = k.render(live=live)
        P, N = torch.from_numpy(pts).cuda(), torch.from_numpy(nrm).cuda()
        shaded = torch.empty((p.rows, p.cols, 4), dtype=torch.uint8, device="cuda")
        tangent = torch.empty_like(shaded)
        capi.check(lib.df_render_image(P.data_ptr(), p.cols * 16, N.data_ptr(), p.cols * 16, p.cols, p.rows, light, shaded.data_ptr(),
                                       p.cols * 4, s))
        capi.check(lib.df_render_tangent_colors(N.data_ptr(), p.cols * 16, p.cols, p.rows, tangent.data_ptr(), p.cols * 4, s))
        shaded, tangent = shaded.cpu().numpy(), tangent.cpu().numpy()
        assert np.array_equal(k.render_image(live=live, flag=0), shaded)
        assert np.array_equal(k.render_image(live=live, flag=1), shaded)
        assert np.array_equal(k.render_image(live=live, flag=2), tangent)
        assert np.array_equal(k.render_image(live=live, flag=3), np.concatenate([shaded, tangent], 1))
        assert len(np.unique(shaded.reshape(-1, 4), axis=0)) > 50
    k.close()


def test_cpp_mirror_renders_the_same_maps(tmp_path):
    from dynamicfusion_b200 import build
    exe = build.build_cpp_program(ROOT / "tests" / "cpp" / "render_export.cpp", ROOT / "tests" / "cpp" / "_build" / "render_export")
    r = subprocess.run([str(exe), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "all checks passed" in r.stdout
    k = kf.KinFu.from_snapshot(tmp_path / "render_export.dfsnap")
    for live, name in ((False, "canonical"), (True, "live")):
        pts, nrm, ids = k.render(live=live)
        assert (ids >= 0).sum() > 1000
        assert (tmp_path / f"{name}_points.bin").read_bytes() == pts.tobytes()
        assert (tmp_path / f"{name}_normals.bin").read_bytes() == nrm.tobytes()
        for flag in (0, 1, 2, 3, 7):
            assert (tmp_path / f"{name}_image{flag}.bin").read_bytes() == k.render_image(live=live, flag=flag).tobytes(), flag
    k.close()


def test_misaligned_pitches_are_refused_without_writing():
    lib = capi.load()
    s = torch.cuda.current_stream().cuda_stream
    cloud, tris, centre, _, _ = sphere_mesh()
    v = torch.from_numpy(cloud).cuda()
    t = torch.from_numpy(np.ascontiguousarray(tris)).cuda()
    cols, rows = 64, 48
    buf = torch.full((rows * (cols + 1) * 4 + 4,), 7.0, dtype=torch.float32, device="cuda")
    ids = torch.full((rows * (cols + 1),), -7, dtype=torch.int32, device="cuda")
    ws = torch.empty(lib.df_raster_workspace_bytes(len(v), len(t), cols, rows), dtype=torch.uint8, device="cuda")
    w2c = capi.make_aff(*look_at(centre, 0.8))
    K = capi.make_intr(*K640)
    for pp, ip in ((cols * 16 + 4, cols * 4), (cols * 16, cols * 4 + 2)):     # not a multiple of 16 / of 4
        st = lib.df_raster_mesh(v.data_ptr(), len(v), 4, t.data_ptr(), len(t), w2c, K, cols, rows, ids.data_ptr(), ip, buf.data_ptr(), pp,
                                buf.data_ptr(), pp, None, ws.data_ptr(), s)
        assert st != 0
    torch.cuda.synchronize()
    assert torch.all(buf == 7.0) and torch.all(ids == -7)
    k = gu.run(gu.kinfu_params(128, 0, max_nodes=1024, cloud_capacity=1_000_000), FRAMES[:4])
    p = k.params
    pts = torch.full((p.rows, p.cols + 1, 4), 7.0, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    st = k.lib.df_kinfu_render(k.h, 0, None, None, 0, pts.data_ptr(), p.cols * 16 + 4, pts.data_ptr(), p.cols * 16 + 4)
    assert st != 0 and torch.all(pts == 7.0)
    k.close()
