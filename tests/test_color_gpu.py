"""Colour on the GPU: df_integrate_color, df_sample_colors and df_mesh_colors equal tests/color_oracle.c bit for bit; the frame loop with
DF_KINFU_COLOR leaves geometry untouched, can be rebuilt from the public entries, resets, resumes from version-2 snapshots, reproduces the
synthetic scene's texture, and exports the same coloured mesh and picture from Python and C++."""
import ctypes as C
import os
import struct
import subprocess
from pathlib import Path

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import color_oracle as co  # noqa: E402
import snapshot_model as sm  # noqa: E402
from dynamicfusion_b200 import build, capi, kinfu as kf, synth  # noqa: E402
import gpu_util as gu  # noqa: E402
from scenes import look_at, sphere_mesh  # noqa: E402

ROOT = Path(__file__).resolve().parents[1]
PARAMS_BYTES = C.sizeof(capi.KinfuParams)


def _random_bgra(rng, rows, cols):
    img = rng.integers(0, 256, (rows, cols, 4), np.uint8)
    img[..., 3] = 255
    return img


# ------------------------------------------------------------------------------------------------------------ df_integrate_color
def _integrate_case(dims, size, cols, rows, depths, pad=0, seed=0):
    """fuse `depths` with random colour images: GPU tracked / dense and oracle tracked / dense colour volumes after every frame"""
    lib = capi.load()
    rng = np.random.default_rng(seed)
    nvox = int(np.prod(dims))
    vs = tuple(size / d for d in dims)
    trunc = max(0.04, 2.1 * max(vs))
    K = synth.scaled_K(cols, rows) if cols != 640 else synth.DEFAULT_K
    intr = capi.make_intr(*K)
    vol2cam = (np.eye(3, dtype=np.float32), np.array([-size / 2, -size / 2, 0.5], np.float32))
    tsdf = torch.zeros(nvox, dtype=torch.int32, device="cuda")
    V = capi.make_volume(tsdf.data_ptr(), dims, vs, trunc, 64)
    act = torch.zeros(lib.df_volume_activity_bytes(V), dtype=torch.uint8, device="cuda")
    g_tr, g_de = (torch.zeros(nvox, dtype=torch.int32, device="cuda") for _ in range(2))
    o_tr, o_de = np.zeros(nvox, np.uint32), np.zeros(nvox, np.uint32)
    visited = []
    for depth in depths:
        d_dev, d_pitch, _ = gu.padded(depth, pad, 0)
        dists = torch.zeros((rows, cols + pad), dtype=torch.int16, device="cuda")
        capi.check(lib.df_compute_dists(d_dev.data_ptr(), d_pitch, cols, rows, intr, dists.data_ptr(), (cols + pad) * 2, gu.stream()))
        capi.check(lib.df_integrate_tracked(V, dists.data_ptr(), (cols + pad) * 2, cols, rows, capi.make_aff(*vol2cam), intr, None,
                                            act.data_ptr(), None, gu.stream()))
        img = _random_bgra(rng, rows, cols)
        i_dev, i_pitch, i_host = gu.padded(img, pad, 99)
        for colours, a in ((g_tr, act.data_ptr()), (g_de, None)):
            capi.check(lib.df_integrate_color(V, colours.data_ptr(), dists.data_ptr(), (cols + pad) * 2, i_dev.data_ptr(), i_pitch, cols, rows,
                                              capi.make_aff(*vol2cam), intr, a, gu.stream()))
        dists_host = dists.cpu().numpy().view(np.uint16)[:, :cols]
        act_host = act.cpu().numpy()
        co.integrate_color(o_tr, dims, vs, trunc, 64, dists_host, i_host, vol2cam, K, act_host)
        co.integrate_color(o_de, dims, vs, trunc, 64, dists_host, i_host, vol2cam, K, None)
        visited.append(float(act_host[:-(-nvox // 1024)].astype(bool).mean()))
        yield g_tr.cpu().numpy().view(np.uint32), g_de.cpu().numpy().view(np.uint32), o_tr, o_de, visited[-1]


@pytest.mark.parametrize("name,dims,size,cols,rows,pad", [("c1_128", (128,) * 3, 3.0, 640, 480, 0), ("c1_256", (256,) * 3, 3.0, 640, 480, 0),
                                                          ("odd_50x40x36", (50, 40, 36), 3.0, 640, 480, 0),
                                                          ("ragged_157x113", (64, 64, 64), 3.0, 157, 113, 5)])
def test_integrate_color_equals_the_oracle(name, dims, size, cols, rows, pad):
    K = synth.scaled_K(cols, rows) if cols != 640 else synth.DEFAULT_K
    depths = [synth.sphere_wall_depth(cols, rows, K, seed=s) for s in range(3)]
    if dims[0] % 4:
        assert name.startswith("odd")                                   # the 1-voxel walk
    n = 0
    for g_tr, g_de, o_tr, o_de, share in _integrate_case(dims, size, cols, rows, depths, pad):
        n += 1
        assert np.array_equal(g_tr, o_tr), (name, n)                    # bit for bit, with the activity map
        assert np.array_equal(g_de, o_de), (name, n)                    # and without
        assert np.array_equal(g_tr, g_de), (name, n)                    # tracked = dense: the band lies inside the marked stretches
        assert 0 < share < 1 or min(dims) < 64
        w = g_tr >> 24
        assert w.max() == n and (w > 0).sum() > 500, (name, n, int(w.max()))
    assert n == 3


# -------------------------------------------------------------------------------------------------------------- df_sample_colors
def _gpu_sample(colours, dims, vs, pose, offset, pts, count=None):
    lib = capi.load()
    P = np.ascontiguousarray(pts, np.float32)
    rows, cols = (1, len(P)) if P.ndim == 2 else P.shape[:2]
    stride = P.shape[-1]
    pd = gu.dev(P)
    out = torch.full((rows, cols), 0x01010101, dtype=torch.int32, device="cuda")
    cnt = None if count is None else torch.tensor([count], dtype=torch.int32, device="cuda")
    V = capi.make_volume(None, dims, vs, 0.04, 64)
    capi.check(lib.df_sample_colors(V, gu.dev(colours).data_ptr(), capi.make_aff(*pose), offset, pd.data_ptr(), cols * stride * 4, stride, cols, rows,
                                    None if cnt is None else cnt.data_ptr(), out.data_ptr(), cols * 4, gu.stream()))
    return out.cpu().numpy().view(np.uint8).reshape(P.shape[:-1] + (4,))


def test_sample_colors_equals_the_oracle():
    dims, size = (128,) * 3, 3.0
    vs = (size / 128,) * 3
    pose = synth.volume_pose(size)
    K = synth.DEFAULT_K
    depths = [synth.sphere_wall_depth(seed=s) for s in range(2)]
    *_, last = _integrate_case(dims, size, 640, 480, depths)
    colours = last[0]
    rng = np.random.default_rng(7)
    coloured = np.flatnonzero(colours >> 24)
    pick = rng.choice(coloured, 200000)
    z, rem = np.divmod(pick, 128 * 128)
    y, x = np.divmod(rem, 128)
    g = np.stack([x, y, z], -1) + rng.uniform(-1.5, 1.5, (len(pick), 3))
    for offset in (0.0, 0.5):
        pts = ((g + offset) * vs[0] + pose[1]).astype(np.float32)
        pts[::97] = np.nan                                              # NaN points
        pts[5::89] *= 40.0                                              # far outside
        pts[7::101, 2] = np.float32(pose[1][2])                         # on the volume's first slice
        want = co.sample_colors(colours, dims, vs, pose, offset, pts)
        got = _gpu_sample(colours, dims, vs, pose, offset, pts)
        assert np.array_equal(got, want)
        assert 0.3 < (want[:, 3] == 255).mean() < 1.0 and not want[::97].any()
        p4 = np.concatenate([pts, np.ones((len(pts), 1), np.float32)], 1)   # float4 points, and a device count that bounds them
        got4 = _gpu_sample(colours, dims, vs, pose, offset, p4, count=1000)
        assert np.array_equal(got4[:1000], want[:1000]) and np.all(got4[1000:] == 1)
    img = ((g[:640 * 100] * vs[0]) + pose[1]).astype(np.float32).reshape(100, 640, 3)   # an image-shaped map
    img4 = np.concatenate([img, np.zeros((100, 640, 1), np.float32)], -1)
    assert np.array_equal(_gpu_sample(colours, dims, vs, pose, 0.0, img4), co.sample_colors(colours, dims, vs, pose, 0.0, img4))


# ---------------------------------------------------------------------------------------------------------------- df_mesh_colors
def _gpu_raster(verts, tris, w2c, K, cols, rows):
    lib = capi.load()
    v, t = gu.dev(np.asarray(verts, np.float32)), gu.dev(np.asarray(tris, np.int32).reshape(-1, 3))
    pts = torch.empty((rows, cols, 4), dtype=torch.float32, device="cuda")
    nrm = torch.empty_like(pts)
    ids = torch.empty((rows, cols), dtype=torch.int32, device="cuda")
    stats = torch.zeros(5, dtype=torch.int64, device="cuda")
    ws = torch.empty(lib.df_raster_workspace_bytes(len(v), len(t), cols, rows), dtype=torch.uint8, device="cuda")
    capi.check(lib.df_raster_mesh(v.data_ptr(), len(v), v.shape[1], t.data_ptr(), len(t), capi.make_aff(*w2c), capi.make_intr(*K), cols, rows,
                                  ids.data_ptr(), cols * 4, pts.data_ptr(), cols * 16, nrm.data_ptr(), cols * 16, stats.data_ptr(), ws.data_ptr(),
                                  gu.stream()))
    return v, t, ids, pts, stats.cpu().numpy()


def _gpu_mesh_colors(v, t, ids, pts, w2c, rgba, cols, rows, pad=3):
    lib = capi.load()
    img = torch.full((rows, cols + pad, 4), 77, dtype=torch.uint8, device="cuda")
    c = gu.dev(np.ascontiguousarray(rgba).view(np.uint32).reshape(-1))
    capi.check(lib.df_mesh_colors(ids.data_ptr(), cols * 4, pts.data_ptr(), cols * 16, v.data_ptr(), len(v), v.shape[1], t.data_ptr(), len(t),
                                  capi.make_aff(*w2c), c.data_ptr(), cols, rows, img.data_ptr(), (cols + pad) * 4, gu.stream()))
    out = img.cpu().numpy()
    assert np.all(out[:, cols:] == 77)                                  # nothing past the image's columns
    return out[:, :cols]


def test_mesh_colors_equals_the_oracle_on_the_sphere():
    cloud, tris, centre, _, _ = sphere_mesh()
    rng = np.random.default_rng(3)
    rgba = rng.integers(0, 256, (len(cloud), 4), np.uint8)
    rgba[:, 3] = 255
    rgba[rng.random(len(cloud)) < 0.2] = 0                              # a fifth of the vertices has no colour
    K = (525.0, 525.0, 319.5, 239.5)
    for name, w2c in (("oblique", look_at(centre, 0.5, (0.3, -0.2, 1.0))), ("close_up", look_at(centre, 0.24, (-0.1, 0.15, 1.0)))):
        v, t, ids, pts, stats = _gpu_raster(cloud, tris, w2c, K, 640, 480)
        if name == "close_up":
            assert stats[3] > 0                                         # the large-triangle path drew some of it
        want = co.mesh_colors(ids.cpu().numpy(), pts.cpu().numpy(), cloud, tris, w2c, rgba)
        got = _gpu_mesh_colors(v, t, ids, pts, w2c, rgba, 640, 480)
        assert np.array_equal(got, want), name
        drawn = ids.cpu().numpy() >= 0
        assert drawn.sum() > 10000 and not got[~drawn].any() and got[drawn][:, :3].any(1).mean() > 0.9


# ------------------------------------------------------------------------------------------------------------------- the frame loop
RGBD = [synth.umbrella_rgbd(t) for t in range(8)]


@pytest.mark.parametrize("extra", [0, kf.LIVE_MODEL, kf.EXTEND_FIELD, kf.RIGID_ONLY], ids=["default", "live_model", "extend_field", "rigid_only"])
def test_colour_never_feeds_back(extra):
    plain, colour = (kf.KinFu(gu.kinfu_params(128, extra, max_nodes=1024, cloud_capacity=1_000_000)),
                     kf.KinFu(gu.kinfu_params(128, extra | kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000)))
    for depth, bgra in RGBD[:6]:
        plain(depth)
        colour(depth, bgra)
        assert colour.info()["launches"] - plain.info()["launches"] == (2 if not (extra & kf.RIGID_ONLY) or colour.info()["frame_counter"] == 1 else 1)
        assert gu.state(plain) == gu.state(colour)
    assert (colour.buffer("color_volume") >> 24).max() == 6
    if not extra & kf.RIGID_ONLY:
        assert (colour.mesh_colors()[:, 3] == 255).mean() > 0.5
    plain.close(); colour.close()


def _rebuild_frame(k, colours, bgra):
    """what the loop did with this frame's colours, from the public entries and the loop's own dists, pose and activity map"""
    lib, p = k.lib, k.params
    ptr, pitch, c_, r_ = C.c_void_p(), C.c_size_t(), C.c_int(), C.c_int()

    def dev_ptr(which):
        capi.check(lib.df_kinfu_get_buffer(k.h, which, C.byref(ptr), C.byref(pitch), C.byref(c_), C.byref(r_)))
        return ptr.value, pitch.value
    vs = tuple(p.volume_size[i] / p.volume_dims[i] for i in range(3))
    V = capi.make_volume(None, tuple(p.volume_dims), vs, max(p.tsdf_trunc_dist, np.float32(2.1) * np.float32(max(vs))), p.tsdf_max_weight)
    vol_pose = (np.array(p.volume_pose.R, np.float32).reshape(3, 3), np.array(p.volume_pose.t, np.float32))
    vol2cam = co.aff_mul(co.aff_inv(k.getCameraPose()), vol_pose)
    dists, dpitch = dev_ptr(kf.BUF["dists"])
    act, _ = dev_ptr(kf.BUF["activity"])
    img = gu.dev(bgra)
    capi.check(lib.df_integrate_color(V, colours.data_ptr(), dists, dpitch, img.data_ptr(), p.cols * 4, p.cols, p.rows, capi.make_aff(*vol2cam),
                                      p.intr, act, gu.stream()))
    cloud, _ = dev_ptr(kf.BUF["cloud"])
    n = k.info()["cloud_points"]
    out = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
    capi.check(lib.df_sample_colors(V, colours.data_ptr(), p.volume_pose, 0.5, cloud, 0, 4, n, 1, None, out.data_ptr(), 0, gu.stream()))
    return out[:n].cpu().numpy().view(np.uint8).reshape(-1, 4)


@pytest.mark.parametrize("overlap", ["1", "0"])
def test_loop_colours_rebuilt_from_the_public_entries(monkeypatch, overlap):
    monkeypatch.setenv("DF_KINFU_OVERLAP_EXTRACT", overlap)
    runs = []
    for rep in range(2):
        k = kf.KinFu(gu.kinfu_params(128, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000))
        mine = torch.zeros(128 ** 3, dtype=torch.int32, device="cuda")
        per_frame = []
        for depth, bgra in RGBD[:5]:
            k(depth, bgra)
            cloud_rgba = _rebuild_frame(k, mine, bgra)
            vol = k.buffer("color_volume")
            assert np.array_equal(vol, mine.cpu().numpy().view(np.uint32))
            assert np.array_equal(k.buffer("cloud_colors"), cloud_rgba) and np.array_equal(k.mesh_colors(), cloud_rgba)
            per_frame.append((vol.tobytes(), cloud_rgba.tobytes()))
        runs.append(per_frame)
        if rep == 1:
            before = (k.buffer("color_volume").copy(), k.state_digest())
            k(RGBD[5][0])                                                # a depth-only frame: geometry moves on, the colour volume stays
            assert np.array_equal(k.buffer("color_volume"), before[0]) and k.state_digest() != before[1]
            assert len(k.mesh_colors()) == k.info()["cloud_points"]
            k.reset()
            assert not k.buffer("color_volume").any()
            k(*RGBD[0])
            assert k.buffer("color_volume").tobytes() == per_frame[0][0]  # and the next first frame starts afresh
        k.close()
    assert runs[0] == runs[1]                                           # two runs, identical


def test_refusals(capfd):
    with pytest.raises(RuntimeError):
        kf.KinFu(gu.kinfu_params(128, kf.COLOR | kf.WARPED_INTEGRATE, max_nodes=1024, cloud_capacity=1_000_000))
    assert "DF_KINFU_WARPED_INTEGRATE" in capfd.readouterr().err
    k = kf.KinFu(gu.kinfu_params(128, 0, max_nodes=1024, cloud_capacity=1_000_000))
    depth, bgra = RGBD[0]
    with pytest.raises(RuntimeError):
        k(depth, bgra)
    with pytest.raises(RuntimeError):
        k(torch.from_numpy(depth.view(np.int16)).cuda(), torch.from_numpy(bgra).cuda())
    assert k.info()["frame_counter"] == 0
    for call in (k.mesh_colors, lambda: k.buffer("color_volume"), lambda: k.render_image(flag=4)):
        with pytest.raises(RuntimeError):
            call()
    k.close()
    k = kf.KinFu(gu.kinfu_params(128, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000))  # device frames give what host frames give
    h = kf.KinFu(gu.kinfu_params(128, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000))
    for depth, bgra in RGBD[:3]:
        k(torch.from_numpy(depth.view(np.int16)).cuda(), torch.from_numpy(bgra).cuda())
        h(depth, bgra)
    assert np.array_equal(k.buffer("color_volume"), h.buffer("color_volume")) and k.state_digest() == h.state_digest()
    k.close(); h.close()


# ------------------------------------------------------------------------------------------------------------------------ fidelity
def test_texture_fidelity_c2_256(tmp_path):
    k = kf.KinFu(gu.kinfu_params(256, kf.COLOR, max_nodes=1024, cloud_capacity=2_000_000))
    for t in range(20):
        k(*synth.umbrella_rgbd(t))
    verts, _, faces = k.mesh()
    rgba = k.mesh_colors()
    # the cap, away from its rim: canonical coordinates are frame 0's world coordinates, where the cap is z = 0.9 + a(0) r^2
    r2 = verts[:, 0] ** 2 + verts[:, 1] ** 2
    cap = (r2 < 0.25 ** 2) & (np.abs(verts[:, 2] - (0.9 + 0.6 * r2)) < 0.05)
    assert cap.sum() > 5000
    coloured = rgba[:, 3] == 255
    frac = coloured[cap].mean()
    err = np.abs(rgba[cap & coloured][:, :3].astype(int) - synth.umbrella_texture(verts[cap & coloured]).astype(int))
    med, p90 = np.median(err), np.percentile(err, 90)
    out = os.environ.get("DF_COLOR_FIDELITY_OUT")
    if out:
        Path(out).write_text(f"cap vertices {int(cap.sum())} coloured fraction {frac:.4f} median {med:.1f} p90 {p90:.1f} "
                             f"all-vertex coloured fraction {coloured.mean():.4f}\n")
    # measured (NVIDIA H100 80GB HBM3, one run): 23,481 cap vertices, all coloured; per-channel error median 12, 90th percentile 51 of 255
    # (the default loop's pose error on this sequence moves the texture by a few millimetres); 94.0 % of all vertices coloured
    assert frac > FIDELITY_MIN_FRACTION and med <= FIDELITY_MEDIAN and p90 <= FIDELITY_P90, (frac, med, p90)
    # the PLY carries these colours
    path = tmp_path / "cap.ply"
    assert k.save_mesh(path, colors=True) == len(faces)
    head, body = path.read_bytes().split(b"end_header\n", 1)
    assert b"property uchar red" in head
    rec = np.frombuffer(body[:27 * len(verts)], np.dtype([("f", "<f4", (6,)), ("c", "u1", (3,))]))
    assert np.array_equal(rec["c"], rgba[:, :3]) and np.array_equal(rec["f"][:, :3], verts)
    # and the picture of the warped model shows the texture
    img = k.render_image(live=True, flag=4)
    ids = k.render(live=True)[2]
    shown = img[ids >= 0][:, :3].any(1).mean()
    assert (ids >= 0).sum() > 50000 and shown > 0.8, shown
    k.close()


FIDELITY_MIN_FRACTION, FIDELITY_MEDIAN, FIDELITY_P90 = 0.9, 20.0, 75.0


# ----------------------------------------------------------------------------------------------------------------------- snapshots
def test_colourless_snapshot_is_version_1():
    k = kf.KinFu(gu.kinfu_params(64, 0, max_nodes=1024, cloud_capacity=1_000_000))
    for depth, _ in RGBD[:3]:
        k(depth)
    snap = k.snapshot()
    magic, version, hlen, total, check = struct.unpack_from("<8sIIQQ", snap)
    assert magic == sm.MAGIC and version == 1 and total == len(snap) and check == sm.checksum(snap[sm.HEADER:])
    cnt = sm.counters(snap, PARAMS_BYTES)
    cls, payload = sm.pack(k.buffer("volume"), (64, 64, 64))
    assert snap.endswith(cls.tobytes() + payload.tobytes()) and cnt[7] == payload.nbytes   # the volume is the last section, as in version 1
    k.close()


def test_version_2_resumes_and_rejects(capfd):
    frames = RGBD[:7]
    ref = kf.KinFu(gu.kinfu_params(64, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000))
    want, snap = [], None
    for i, (depth, bgra) in enumerate(frames):
        ref(depth, bgra)
        want.append((ref.state_digest(), ref.buffer("color_volume").tobytes(), ref.buffer("cloud_colors").tobytes()))
        if i == 3:
            snap = ref.snapshot()
    ref.close()
    assert struct.unpack_from("<I", snap, 8)[0] == 2
    n_cloud = sm.counters(snap, PARAMS_BYTES)[4]
    assert kf.KinFu.snapshot_params(snap).flags & kf.COLOR
    k = kf.KinFu(gu.kinfu_params(64, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000))
    k(*frames[0])
    before = (k.state_digest(), k.buffer("color_volume").tobytes(), k.buffer("cloud_colors").tobytes())
    # damaged colour sections are refused with the state unchanged
    cls_at = len(snap) - 4 * n_cloud
    bad = []
    bad.append(sm.header(snap[sm.HEADER:-4], version=2) + snap[sm.HEADER:-4])             # truncated
    flip = bytearray(snap); flip[cls_at - 5] ^= 0x10                                       # payload bit, checksum stale
    bad.append(bytes(flip))
    body = bytearray(snap[sm.HEADER:])
    nb = sm.brick_count((64, 64, 64))
    # where version 1 ends (the format's section lengths, dfusion.h) the colour length word begins
    cnt = sm.counters(snap, PARAMS_BYTES)
    prm = k.params
    act = k.lib.df_volume_activity_bytes(capi.make_volume(None, (64, 64, 64), (1.0,) * 3, 0.04, 64))
    pyr = sum((prm.cols >> l) * (prm.rows >> l) * 32 for l in range(3))
    clen_at = PARAMS_BYTES + sm.F2_BYTES + sm.COUNTERS.size + cnt[5] * 48 + cnt[3] * 48 + act + pyr + n_cloud * 32 + nb + cnt[7]
    assert clen_at + 8 + nb + struct.unpack_from("<Q", body, clen_at)[0] + 4 * n_cloud == len(body)
    wrong = bytearray(body); wrong[clen_at + 8] = 3                                        # a class byte outside {0, 1, 2}, resealed
    bad.append(sm.header(bytes(wrong), version=2) + bytes(wrong))
    for b in bad:
        with pytest.raises(RuntimeError):
            k.restore(b)
        assert (k.state_digest(), k.buffer("color_volume").tobytes(), k.buffer("cloud_colors").tobytes()) == before
    assert "rejected" in capfd.readouterr().err
    plain = kf.KinFu(gu.kinfu_params(64, 0, max_nodes=1024, cloud_capacity=1_000_000))
    with pytest.raises(RuntimeError):
        plain.restore(snap)                                             # other parameters
    plain.close()
    k.restore(snap)
    assert (k.state_digest(), k.buffer("color_volume").tobytes(), k.buffer("cloud_colors").tobytes()) == want[3]
    for i in range(4, 7):
        k(*frames[i])
        assert (k.state_digest(), k.buffer("color_volume").tobytes(), k.buffer("cloud_colors").tobytes()) == want[i]
    k.close()


# --------------------------------------------------------------------------------------------------------------------------- hosts
def test_render_image_flag_4_is_mesh_colors_of_the_render():
    k = kf.KinFu(gu.kinfu_params(128, kf.COLOR, max_nodes=1024, cloud_capacity=1_000_000))
    for depth, bgra in RGBD[:6]:
        k(depth, bgra)
    digest = k.state_digest()
    for live in (False, True):
        img = k.render_image(live=live, flag=4)
        pts, _, ids = k.render(live=live)
        verts, _, faces = k.mesh(live=live)
        R, t = (np.eye(3, dtype=np.float32), np.zeros(3, np.float32)) if live else k.getCameraPose()
        want = co.mesh_colors(ids, pts, verts, faces, co.aff_inv((R, t)), k.mesh_colors())
        assert np.array_equal(img, want), live
        assert img[ids >= 0][:, :3].any(1).mean() > 0.5
    assert k.state_digest() == digest
    k.close()


def test_cpp_mirror_exports_the_same_colours(tmp_path):
    exe = build.build_cpp_program(ROOT / "tests" / "cpp" / "color_export.cpp", ROOT / "tests" / "cpp" / "_build" / "color_export")
    frames = RGBD[:5]
    np.stack([d for d, _ in frames]).tofile(tmp_path / "depth.u16")
    np.stack([c for _, c in frames]).tofile(tmp_path / "bgra.u8")
    r = subprocess.run([str(exe), str(tmp_path / "depth.u16"), str(tmp_path / "bgra.u8"), str(len(frames)), str(tmp_path / "cpp.ply"),
                        str(tmp_path / "cpp.bgra")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    p = kf.KinFuParams.default_params_dynamicfusion()
    p.flags = kf.COLOR
    k = kf.KinFu(p)
    for depth, bgra in frames:
        k(depth, bgra)
    k.save_mesh(tmp_path / "py.ply", live=True, colors=True)
    img = k.render_image(live=True, flag=4)
    k.close()
    assert (tmp_path / "cpp.ply").read_bytes() == (tmp_path / "py.ply").read_bytes()
    assert (tmp_path / "cpp.bgra").read_bytes() == img.tobytes()
