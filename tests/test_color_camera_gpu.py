"""The colour camera on the GPU: df_color_depth_map and df_integrate_color_camera equal tests/color_camera_oracle.c bit for bit; the
occlusion test keeps the small sphere's colour off the wall behind it; the frame loop with a colour camera leaves geometry untouched, can
be rebuilt from the public entries, resets, refuses what it must, resumes from version-3 snapshots, reproduces the synthetic scene's texture
through a Kinect-v2-like camera, and exports the same coloured mesh and picture from Python and C++."""
import ctypes as C
import functools
import os
import struct
import subprocess
from pathlib import Path

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import color_camera_oracle as cco  # noqa: E402
import color_oracle as co  # noqa: E402
import snapshot_model as sm  # noqa: E402
from dynamicfusion_b200 import build, capi, kinfu as kf, synth  # noqa: E402
import gpu_util as gu  # noqa: E402

ROOT = Path(__file__).resolve().parents[1]
I3 = np.eye(3, dtype=np.float32)


def _rot(deg_y):
    a = np.deg2rad(deg_y)
    return np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]], np.float32)


def _cam_struct(cam: cco.Camera):
    return capi.make_color_camera(cam.K, cam.cols, cam.rows, cam.d2c)


# ------------------------------------------------------------------------------------------------------- both kernels against the oracle
BIG = ((1620.0, 1620.0, 959.5, 539.5), 1920, 1080)          # 1920 x 1080, cell 3 against the 570-pixel depth camera
SMALL = ((285.171, 285.171, 159.5, 119.5), 320, 240)         # 320 x 240, cell 1
D2C = (_rot(1.5), np.array([-0.05, 0.004, 0.002], np.float32))


def _kernel_case(dims, size, cols, rows, K, depths, cam, pad, cpad, seed=0):
    """fuse `depths` with random colour-camera images: per frame (GPU map, oracle map, GPU tracked / dense, oracle tracked / dense)"""
    lib = capi.load()
    rng = np.random.default_rng(seed)
    nvox = int(np.prod(dims))
    vs = tuple(size / d for d in dims)
    trunc = max(0.04, 2.1 * max(vs))
    intr = capi.make_intr(*K)
    vol2cam = (I3, np.array([-size / 2, -size / 2, 0.5], np.float32))
    tsdf = torch.zeros(nvox, dtype=torch.int32, device="cuda")
    V = capi.make_volume(tsdf.data_ptr(), dims, vs, trunc, 64)
    act = torch.zeros(lib.df_volume_activity_bytes(V), dtype=torch.uint8, device="cuda")
    g_tr, g_de = (torch.zeros(nvox, dtype=torch.int32, device="cuda") for _ in range(2))
    o_tr, o_de = np.zeros(nvox, np.uint32), np.zeros(nvox, np.uint32)
    mc, mr, _ = cco.map_dims(K, cam)
    cs = _cam_struct(cam)
    for depth in depths:
        d_dev, d_pitch, d_host = gu.padded(depth, pad, 7)
        dists = torch.zeros((rows, cols + pad), dtype=torch.int16, device="cuda")
        capi.check(lib.df_compute_dists(d_dev.data_ptr(), d_pitch, cols, rows, intr, dists.data_ptr(), (cols + pad) * 2, gu.stream()))
        capi.check(lib.df_integrate_tracked(V, dists.data_ptr(), (cols + pad) * 2, cols, rows, capi.make_aff(*vol2cam), intr, None,
                                            act.data_ptr(), None, gu.stream()))
        cmap = torch.full((mr, mc + cpad), 0x5a5a5a5a, dtype=torch.int32, device="cuda")
        capi.check(lib.df_color_depth_map(d_dev.data_ptr(), d_pitch, cols, rows, intr, cs, cmap.data_ptr(), (mc + cpad) * 4, gu.stream()))
        img = rng.integers(0, 256, (cam.rows, cam.cols, 4), np.uint8)
        i_dev, i_pitch, i_host = gu.padded(img, cpad, 99)
        for colours, a in ((g_tr, act.data_ptr()), (g_de, None)):
            capi.check(lib.df_integrate_color_camera(V, colours.data_ptr(), dists.data_ptr(), (cols + pad) * 2, cols, rows, capi.make_aff(*vol2cam),
                                                     intr, cs, i_dev.data_ptr(), i_pitch, cmap.data_ptr(), (mc + cpad) * 4, a, gu.stream()))
        gmap = cmap.cpu().numpy().view(np.uint32)
        assert np.all(gmap[:, mc:] == 0x5a5a5a5a)                      # nothing written past the map's columns
        omap = cco.depth_map(d_host, K, cam)
        dists_host = dists.cpu().numpy().view(np.uint16)[:, :cols]
        act_host = act.cpu().numpy()
        cco.integrate_color_camera(o_tr, dims, vs, trunc, 64, dists_host, vol2cam, K, cam, i_host, omap, act_host)
        cco.integrate_color_camera(o_de, dims, vs, trunc, 64, dists_host, vol2cam, K, cam, i_host, omap, None)
        yield gmap[:, :mc], omap, g_tr.cpu().numpy().view(np.uint32), g_de.cpu().numpy().view(np.uint32), o_tr, o_de


@pytest.mark.parametrize("name,dims,size,cols,rows,pad,camera,cpad", [
    ("c1_128_big", (128,) * 3, 3.0, 640, 480, 0, BIG, 0),
    ("c1_128_small", (128,) * 3, 3.0, 640, 480, 0, SMALL, 4),
    ("c2_128_big", (128,) * 3, 1.0, 640, 480, 0, BIG, 2),
    ("c2_128_small", (128,) * 3, 1.0, 640, 480, 0, SMALL, 0),
    ("odd_50x40x36", (50, 40, 36), 3.0, 640, 480, 0, SMALL, 0),
    ("ragged_157x113", (64, 64, 64), 3.0, 157, 113, 5, ((120.0, 131.0, 104.5, 47.0), 211, 97), 3)])
def test_kernels_equal_the_oracle(name, dims, size, cols, rows, pad, camera, cpad):
    K = synth.scaled_K(cols, rows) if cols != 640 else synth.DEFAULT_K
    if name.startswith("c2"):
        depths = [synth.umbrella_depth(t) for t in range(3)]
    else:
        depths = [synth.sphere_wall_depth(cols, rows, K, seed=s) for s in range(3)]
    cam = cco.Camera(camera[1], camera[2], camera[0], D2C)
    if dims[0] % 4:
        assert name.startswith("odd")                                   # the 1-voxel walk
    n = 0
    for gmap, omap, g_tr, g_de, o_tr, o_de in _kernel_case(dims, size, cols, rows, K, depths, cam, pad, cpad):
        n += 1
        assert np.array_equal(gmap, omap), (name, n)
        assert np.array_equal(g_tr, o_tr), (name, n)                    # bit for bit, with the activity map
        assert np.array_equal(g_de, o_de), (name, n)                    # and without
        assert np.array_equal(g_tr, g_de), (name, n)
        assert 0.2 < (omap != cco.EMPTY).mean() <= 1.0, (name, n)
        w = g_tr >> 24
        assert w.max() == n and (w > 0).sum() > 300, (name, n, int(w.max()))
    assert n == 3


# ------------------------------------------------------------------------------------------------------------------------ occlusion
SPHERE_C, SPHERE_R = np.array([0.27, -0.17, 1.02]), 0.07


def _segment_distance(a, b, c):
    """distance from point c to the segments a -> b (b: [..., 3]) and the segment parameter of the closest point"""
    d = b - a
    s = np.clip(((c - a) * d).sum(-1) / (d * d).sum(-1), 0.0, 1.0)
    return np.linalg.norm(a + s[..., None] * d - c, axis=-1), s


def _raw(k, which):
    ptr, pitch, c_, r_ = C.c_void_p(), C.c_size_t(), C.c_int(), C.c_int()
    capi.check(k.lib.df_kinfu_get_buffer(k.h, which, C.byref(ptr), C.byref(pitch), C.byref(c_), C.byref(r_)))
    out = np.empty(pitch.value * r_.value, np.uint8)
    capi.check(k.lib.df_kinfu_read_buffer(k.h, which, out.ctypes.data, out.nbytes))
    return out


def test_occlusion_keeps_the_sphere_off_the_wall():
    centre = np.array([-0.1, 0.0, 0.0])                                # the colour camera 0.1 m to the depth camera's -x: its view of the
    Kc = (1081.37, 1081.37, 959.5, 539.5)                               # wall behind the small sphere is blocked further out, off the cap
    cam = cco.Camera(1920, 1080, Kc, (I3, (-centre).astype(np.float32)))
    depth, bgra = synth.umbrella_rgbd(0, color_camera=(Kc, 1920, 1080, cam.d2c))
    k = kf.KinFu(gu.kinfu_params(128, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000))
    k.set_color_camera(Kc, 1920, 1080, cam.d2c)
    k(depth, bgra)
    loop = k.buffer("color_volume")
    # the same frame with a map that hides nothing (every word the largest finite float)
    p = k.params
    vs = tuple(p.volume_size[i] / p.volume_dims[i] for i in range(3))
    trunc = max(p.tsdf_trunc_dist, np.float32(2.1) * np.float32(max(vs)))
    vol_pose = (np.array(p.volume_pose.R, np.float32).reshape(3, 3), np.array(p.volume_pose.t, np.float32))
    vol2cam = co.aff_mul(co.aff_inv(k.getCameraPose()), vol_pose)
    mc, mr, _ = cco.map_dims(synth.DEFAULT_K, cam)
    open_map = np.full((mr, mc), 0x7F7FFFFF, np.uint32)
    dists, act = k.buffer("dists"), _raw(k, kf.BUF["activity"])
    free = cco.integrate_color_camera(np.zeros_like(loop), tuple(p.volume_dims), vs, trunc, p.tsdf_max_weight, dists, vol2cam, synth.DEFAULT_K, cam,
                                      bgra, open_map, act)
    # the oracle with the loop's own map reproduces the loop
    assert np.array_equal(cco.integrate_color_camera(np.zeros_like(loop), tuple(p.volume_dims), vs, trunc, p.tsdf_max_weight, dists, vol2cam,
                                                     synth.DEFAULT_K, cam, bgra, k.buffer("color_map"), act), loop)
    # wall voxels the sphere hides from the colour camera but not from the depth camera, found analytically (frame 0: world = camera)
    D = p.volume_dims[0]
    z, y, x = np.meshgrid(np.arange(D), np.arange(D), np.arange(D), indexing="ij")
    pts = np.stack([x, y, z], -1).reshape(-1, 3) * vs[0] + vol_pose[1].astype(np.float64)
    n = np.array([-0.10, -0.05, 1.0])
    on_wall = np.abs((pts - np.array([0.0, 0.0, 1.3])) @ n / np.linalg.norm(n)) < 0.02
    seen_c, s_c = _segment_distance(centre, pts, SPHERE_C)
    seen_d, _ = _segment_distance(np.zeros(3), pts, SPHERE_C)
    hidden = on_wall & (seen_c < SPHERE_R - 0.005) & (s_c < 0.95) & (seen_d > SPHERE_R + 0.005)

    def red(vol):
        rgb = np.stack([vol & 0xFF, (vol >> 8) & 0xFF, (vol >> 16) & 0xFF], -1).astype(int)
        return ((vol >> 24) > 0) & (np.abs(rgb - np.array(synth.SPHERE_RGB)).max(-1) <= 40)
    print(f"hidden wall voxels {int(hidden.sum())}, coloured by the loop {int((hidden & (loop >> 24 > 0)).sum())}, red without occlusion "
          f"{int((hidden & red(free)).sum())}, red in the loop {int((hidden & red(loop)).sum())}")
    # measured (CPU oracle on the same inputs): 225 hidden wall voxels, 203 of them red without the occlusion test, none with it
    assert hidden.sum() > 100 and (hidden & red(free)).sum() > 100      # the scene does test the rule
    assert not (hidden & red(loop)).any()
    k.close()


# ------------------------------------------------------------------------------------------------------------------- the frame loop
KV2 = ((1081.37, 1081.37, 959.5, 539.5), 1920, 1080, (I3, np.array([-0.052, 0.0, 0.0], np.float32)))   # Kinect-v2-like, 52 mm baseline


@functools.lru_cache(maxsize=None)
def _frame(t):
    return synth.umbrella_rgbd(t, color_camera=KV2)


def _frames(n):
    return [_frame(t) for t in range(n)]


def _with_camera(p, camera=KV2):
    k = kf.KinFu(p)
    k.set_color_camera(camera[0], camera[1], camera[2], camera[3])
    return k


@pytest.mark.parametrize("extra", [0, kf.LIVE_MODEL, kf.EXTEND_FIELD, kf.RIGID_ONLY], ids=["default", "live_model", "extend_field", "rigid_only"])
def test_colour_camera_never_feeds_back(extra):
    plain, colour = (kf.KinFu(gu.kinfu_params(128, extra, max_nodes=1024, cloud_capacity=1_000_000)),
                     _with_camera(gu.kinfu_params(128, extra | kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000)))
    for depth, bgra in _frames(6):
        plain(depth)
        colour(depth, bgra)
        first = colour.info()["frame_counter"] == 1
        assert colour.info()["launches"] - plain.info()["launches"] == (3 if not (extra & kf.RIGID_ONLY) or first else 2)
        assert gu.state(plain) == gu.state(colour)
    assert (colour.buffer("color_volume") >> 24).max() == 6
    if not extra & kf.RIGID_ONLY:
        assert (colour.mesh_colors()[:, 3] == 255).mean() > 0.5
    plain.close(); colour.close()


def _rebuild_frame(k, colours, depth, bgra, cam):
    """the loop's map and this frame's colours from the public entries, with the loop's own dists, pose and activity map"""
    lib, p = k.lib, k.params
    ptr, pitch, c_, r_ = C.c_void_p(), C.c_size_t(), C.c_int(), C.c_int()

    def dev_ptr(which):
        capi.check(lib.df_kinfu_get_buffer(k.h, which, C.byref(ptr), C.byref(pitch), C.byref(c_), C.byref(r_)))
        return ptr.value, pitch.value
    cs = _cam_struct(cam)
    mc, mr, _ = cco.map_dims(synth.DEFAULT_K, cam)
    cmap = torch.zeros((mr, mc), dtype=torch.int32, device="cuda")
    d_dev = gu.dev(depth)
    capi.check(lib.df_color_depth_map(d_dev.data_ptr(), p.cols * 2, p.cols, p.rows, p.intr, cs, cmap.data_ptr(), mc * 4, gu.stream()))
    vs = tuple(p.volume_size[i] / p.volume_dims[i] for i in range(3))
    V = capi.make_volume(None, tuple(p.volume_dims), vs, max(p.tsdf_trunc_dist, np.float32(2.1) * np.float32(max(vs))), p.tsdf_max_weight)
    vol_pose = (np.array(p.volume_pose.R, np.float32).reshape(3, 3), np.array(p.volume_pose.t, np.float32))
    vol2cam = co.aff_mul(co.aff_inv(k.getCameraPose()), vol_pose)
    dists, dpitch = dev_ptr(kf.BUF["dists"])
    act, _ = dev_ptr(kf.BUF["activity"])
    img = gu.dev(bgra)
    capi.check(lib.df_integrate_color_camera(V, colours.data_ptr(), dists, dpitch, p.cols, p.rows, capi.make_aff(*vol2cam), p.intr, cs, img.data_ptr(),
                                             cam.cols * 4, cmap.data_ptr(), mc * 4, act, gu.stream()))
    cloud, _ = dev_ptr(kf.BUF["cloud"])
    n = k.info()["cloud_points"]
    out = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
    capi.check(lib.df_sample_colors(V, colours.data_ptr(), p.volume_pose, 0.5, cloud, 0, 4, n, 1, None, out.data_ptr(), 0, gu.stream()))
    return cmap.cpu().numpy().view(np.uint32), out[:n].cpu().numpy().view(np.uint8).reshape(-1, 4)


@pytest.mark.parametrize("overlap", ["1", "0"])
def test_loop_rebuilt_from_the_public_entries(monkeypatch, overlap):
    monkeypatch.setenv("DF_KINFU_OVERLAP_EXTRACT", overlap)
    cam = cco.Camera(KV2[1], KV2[2], KV2[0], KV2[3])
    runs = []
    for rep in range(2):
        k = _with_camera(gu.kinfu_params(128, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000))
        mine = torch.zeros(128 ** 3, dtype=torch.int32, device="cuda")
        per_frame = []
        for depth, bgra in _frames(5):
            k(depth, bgra)
            cmap, cloud_rgba = _rebuild_frame(k, mine, depth, bgra, cam)
            assert np.array_equal(k.buffer("color_map"), cmap)
            vol = k.buffer("color_volume")
            assert np.array_equal(vol, mine.cpu().numpy().view(np.uint32))
            assert np.array_equal(k.buffer("cloud_colors"), cloud_rgba) and np.array_equal(k.mesh_colors(), cloud_rgba)
            per_frame.append((cmap.tobytes(), vol.tobytes(), cloud_rgba.tobytes()))
        runs.append(per_frame)
        if rep == 1:
            k.reset()                                                   # reset keeps the camera and clears the volume
            assert not k.buffer("color_volume").any() and k.buffer("color_map").shape == cmap.shape
            k(*_frames(1)[0])
            assert (k.buffer("color_map").tobytes(), k.buffer("color_volume").tobytes()) == per_frame[0][:2]
        k.close()
    assert runs[0] == runs[1]                                           # two runs, identical


def test_identity_camera_agrees_with_the_registered_path():
    """a colour camera equal to the depth camera: the same pixels, only the occlusion map's coverage differs"""
    reg, idc = (kf.KinFu(gu.kinfu_params(128, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000)),
                _with_camera(gu.kinfu_params(128, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000),
                             (synth.DEFAULT_K, 640, 480, (I3, np.zeros(3, np.float32)))))
    for t in range(6):
        depth, bgra = synth.umbrella_rgbd(t)
        reg(depth, bgra)
        idc(depth, bgra)
    a, b = reg.buffer("color_volume"), idc.buffer("color_volume")
    either = ((a >> 24) > 0) | ((b >> 24) > 0)
    share = float((a[either] == b[either]).mean())
    print(f"identity camera: {int(either.sum())} coloured voxels, {share:.4f} equal to the registered path")
    # measured (NVIDIA H100 80GB HBM3, one run, 6 frames at 128^3): 61,943 coloured voxels, 81.7 % of them equal.  The rest differ because
    # at cell 1 a depth pixel reprojected and projected again can land one pixel over (the floor of i - ulp), leaving some cells of the
    # occlusion map empty; a voxel seen through an empty cell skips that frame's sample.  The camera never colours a voxel the registered
    # path leaves uncoloured.
    assert share >= IDENTITY_MIN_SHARE and not (((b >> 24) > 0) & ((a >> 24) == 0)).any()
    reg.close(); idc.close()


IDENTITY_MIN_SHARE = 0.8


def test_texture_fidelity_c2_256_kinect_v2_camera():
    k = _with_camera(gu.kinfu_params(256, kf.COLOR, max_nodes=1024, cloud_capacity=2_000_000))
    for depth, bgra in _frames(20):
        k(depth, bgra)
    verts, _, faces = k.mesh()
    rgba = k.mesh_colors()
    r2 = verts[:, 0] ** 2 + verts[:, 1] ** 2
    cap = (r2 < 0.25 ** 2) & (np.abs(verts[:, 2] - (0.9 + 0.6 * r2)) < 0.05)
    assert cap.sum() > 5000
    coloured = rgba[:, 3] == 255
    frac = coloured[cap].mean()
    err = np.abs(rgba[cap & coloured][:, :3].astype(int) - synth.umbrella_texture(verts[cap & coloured]).astype(int))
    med, p90 = np.median(err), np.percentile(err, 90)
    line = (f"cap vertices {int(cap.sum())} coloured fraction {frac:.4f} median {med:.1f} p90 {p90:.1f} "
            f"all-vertex coloured fraction {coloured.mean():.4f}")
    print(line)
    out = os.environ.get("DF_COLOR_FIDELITY_OUT")
    if out:
        Path(out).write_text(line + "\n")
    # measured (NVIDIA H100 80GB HBM3, one run): 23,481 cap vertices, all coloured; per-channel error median 13, 90th percentile 52 of 255;
    # 92.7 % of all vertices coloured (the registered path on the same frames: median 12, 90th percentile 51, 94.0 %)
    assert frac > 0.9 and med <= 20 and p90 <= 75, (frac, med, p90)
    k.close()


# ------------------------------------------------------------------------------------------------------------------------- refusals
def test_refusals_write_nothing(capfd):
    depth, bgra = _frames(1)[0]
    plain = kf.KinFu(gu.kinfu_params(128, 0, max_nodes=1024, cloud_capacity=1_000_000))
    with pytest.raises(RuntimeError):
        plain.set_color_camera(*KV2)                                    # no colour volume
    plain.close()
    k = kf.KinFu(gu.kinfu_params(128, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000))
    with pytest.raises(RuntimeError):
        k.set_color_camera((0.0, 1081.0, 959.5, 539.5), 1920, 1080)     # invalid intrinsics
    with pytest.raises(RuntimeError):
        k.set_color_camera(KV2[0], 0, 1080)
    with pytest.raises(RuntimeError):
        k.buffer("color_map")                                           # still no camera: no map
    k.set_color_camera(*KV2)
    with pytest.raises(ValueError):
        k(depth, synth.umbrella_rgbd(0)[1])                             # an image of the depth's size
    lib = k.lib
    r = lib.df_kinfu_process_host_color(k.h, depth.ctypes.data, depth.strides[0], bgra.ctypes.data, 1919 * 4)   # a pitch below the width
    assert r < 0 and k.info()["frame_counter"] == 0 and not k.buffer("color_volume").any()
    k(depth, bgra)
    before = (k.state_digest(), k.buffer("color_volume").tobytes(), k.buffer("color_map").tobytes())
    with pytest.raises(RuntimeError):
        k.set_color_camera(*KV2)                                        # after frame 0
    with pytest.raises(RuntimeError):
        k.set_color_camera(None)
    assert (k.state_digest(), k.buffer("color_volume").tobytes(), k.buffer("color_map").tobytes()) == before
    k.reset()
    k.set_color_camera(None)                                            # back to registered images once the counter is 0
    with pytest.raises(RuntimeError):
        k.buffer("color_map")
    d, c = synth.umbrella_rgbd(0)
    k(d, c)
    assert (k.buffer("color_volume") >> 24).max() == 1
    k.close()


def test_version_3_resumes_and_rejects(tmp_path, capfd):
    frames = _frames(7)
    ref = _with_camera(gu.kinfu_params(64, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000))
    want, snap = [], None
    for i, (depth, bgra) in enumerate(frames):
        ref(depth, bgra)
        want.append((ref.state_digest(), ref.buffer("color_volume").tobytes(), ref.buffer("cloud_colors").tobytes()))
        if i == 3:
            snap = ref.snapshot()
    ref.close()
    assert struct.unpack_from("<I", snap, 8)[0] == 3
    assert bytes(kf.KinFu.snapshot_color_camera(snap)) == bytes(_cam_struct(cco.Camera(KV2[1], KV2[2], KV2[0], KV2[3])))
    assert snap[-72:] == bytes(kf.KinFu.snapshot_color_camera(snap))
    # an object without a camera, or with another one, refuses it and keeps its state; a version-2 snapshot is refused by a camera object
    other = _with_camera(gu.kinfu_params(64, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000),
                         (KV2[0], 1920, 1080, (I3, np.array([-0.05, 0.0, 0.0], np.float32))))
    none = kf.KinFu(gu.kinfu_params(64, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000))
    d0, c0 = synth.umbrella_rgbd(0)
    none(d0, c0)
    none_snap = none.snapshot()
    assert struct.unpack_from("<I", none_snap, 8)[0] == 2
    for obj in (other, none):
        before = (obj.state_digest(), obj.buffer("color_volume").tobytes())
        with pytest.raises(RuntimeError):
            obj.restore(snap)
        assert (obj.state_digest(), obj.buffer("color_volume").tobytes()) == before
    fresh = _with_camera(gu.kinfu_params(64, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000))
    with pytest.raises(RuntimeError):
        fresh.restore(none_snap)
    assert "colour camera differs" in capfd.readouterr().err
    other.close(); none.close(); fresh.close()
    # resume through a file: from_snapshot sets the camera before loading
    path = tmp_path / "v3.dfsnap"
    path.write_bytes(snap)
    k = kf.KinFu.from_snapshot(path)
    assert k.color_camera is not None and (k.color_camera.cols, k.color_camera.rows) == (1920, 1080)
    assert (k.state_digest(), k.buffer("color_volume").tobytes(), k.buffer("cloud_colors").tobytes()) == want[3]
    for i in range(4, 7):
        k(*frames[i])
        assert (k.state_digest(), k.buffer("color_volume").tobytes(), k.buffer("cloud_colors").tobytes()) == want[i]
    assert k.snapshot()[:8] == sm.MAGIC
    k.close()


# --------------------------------------------------------------------------------------------------------------------------- hosts
def test_cpp_mirror_exports_the_same_colours(tmp_path):
    exe = build.build_cpp_program(ROOT / "tests" / "cpp" / "color_camera_export.cpp", ROOT / "tests" / "cpp" / "_build" / "color_camera_export")
    frames = _frames(5)
    np.stack([d for d, _ in frames]).tofile(tmp_path / "depth.u16")
    np.stack([c for _, c in frames]).tofile(tmp_path / "bgra.u8")
    K, cols, rows, (R, t) = KV2
    nums = [repr(float(np.float32(x))) for x in list(K) + list(np.asarray(R).reshape(9)) + list(t)]
    r = subprocess.run([str(exe), str(tmp_path / "depth.u16"), str(tmp_path / "bgra.u8"), str(len(frames)), str(cols), str(rows), *nums,
                        str(tmp_path / "cpp.ply"), str(tmp_path / "cpp.bgra")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    p = kf.KinFuParams.default_params_dynamicfusion()
    p.flags = kf.COLOR
    k = _with_camera(p)
    for depth, bgra in frames:
        k(depth, bgra)
    k.save_mesh(tmp_path / "py.ply", live=True, colors=True)
    img = k.render_image(live=True, flag=4)
    k.close()
    assert (tmp_path / "cpp.ply").read_bytes() == (tmp_path / "py.ply").read_bytes()
    assert (tmp_path / "cpp.bgra").read_bytes() == img.tobytes()
