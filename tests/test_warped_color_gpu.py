"""Colour under per-voxel warped fusion on the GPU.  df_integrate_warped_color (csrc/fusion.cu) against df_integrate_warped and the oracle
(tests/warped_color_oracle.c over oracle/orc_fusion.c) in its three modes -- registered image, colour camera, colour camera through a lens:
the TSDF volume, activity map and counters are df_integrate_warped's bit for bit, and the colour words are the oracle's except where the TSDF
side already differs from the oracle within test_fusion_gpu.py's 1e-5 budget (the double exp() of the node weights).  Then the frame loop
with DF_KINFU_WARPED_COLOR: colour never feeds back, the loop's colour volume is rebuilt frame by frame from the public entries, depth-only
frames leave it alone, a snapshot resumes exactly, the flag is refused without its two companions, and colour tracking runs with it."""
import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import color_camera_oracle as cco  # noqa: E402
import color_oracle as co  # noqa: E402
import gpu_util as gu  # noqa: E402
import lens_oracle as lo  # noqa: E402
import warped_color_oracle as wco  # noqa: E402
from dynamicfusion_b200 import build, capi, host, synth  # noqa: E402
from dynamicfusion_b200 import kinfu as kf  # noqa: E402
from warp_cases import K, MAXW, _surface_nodes, _tilted_pose, _volume  # noqa: E402

ROOT = Path(__file__).resolve().parents[1]
MODES = ["registered", "camera", "camera_lens"]
LENS = (0.08, -0.03, 0.001, -0.0005, 0.0, 0.0, 0.0, 0.0)


def _camera(mode, cols, rows, scale=1.5):
    if mode == "registered":
        return None, None
    ccols, crows = int(cols * scale), int(rows * scale)
    cam = cco.Camera(ccols, crows, (K[0] * scale, K[1] * scale, ccols / 2.0, crows / 2.0),
                     (np.eye(3, dtype=np.float32), np.array([0.025, -0.004, 0.002], np.float32)))
    lens = capi.make_lens(LENS, K=cam.K, cols=ccols, rows=crows) if mode == "camera_lens" else None
    return cam, lens


def _run_modes(orc, vol_factory, depth, nodes, cam_pose, weight_scale, mode, pad=0, scale=1.5, seed=0):
    """df_integrate_warped and df_integrate_warped_color on the same inputs, and the oracle: (plain, coloured, oracle) dicts"""
    rows, cols = depth.shape
    cam, lens = _camera(mode, cols, rows, scale)
    rng = np.random.default_rng(seed)
    ish = (rows, cols) if cam is None else (cam.rows, cam.cols)
    bgra = rng.integers(0, 256, ish + (4,), dtype=np.uint8)
    img_dev, img_pitch, img_host = gu.padded(bgra, pad, 0)
    cmap = cmap_dev = None
    if cam is not None:
        cmap = lo.depth_map(depth, K, cam, lens)
        cmap_dev = gu.dev(cmap)
    wf = host.WarpField()
    wf.setNodes(torch.from_numpy(nodes).cuda())
    d_depth = host.u16_to_device(depth)
    plain, coloured = vol_factory(), vol_factory()
    nvox = int(np.prod(plain.getDims()))
    c_plain = torch.zeros(2, dtype=torch.int64, device="cuda")
    c_col = torch.zeros(3, dtype=torch.int64, device="cuda")
    colours = torch.zeros(nvox, dtype=torch.int32, device="cuda")
    world2cam = plain.integrate_warped(d_depth, cam_pose, K, wf, weight_scale, c_plain)
    ccam = None if cam is None else capi.make_color_camera(cam.K, cam.cols, cam.rows, cam.d2c)
    lib = capi.load()
    capi.check(lib.df_integrate_warped_color(
        coloured._vol(), d_depth.data_ptr(), cols * 2, cols, rows, capi.make_aff(*coloured.pose_), capi.make_aff(*world2cam), capi.make_intr(*K),
        wf.nodes_.data_ptr(), wf.nodes_.shape[0], wf.grid_.data_ptr(), float(weight_scale), c_col.data_ptr(), coloured.activity_.data_ptr(), None,
        colours.data_ptr(), img_dev.data_ptr(), img_pitch, C.byref(ccam) if ccam is not None else None,
        C.byref(lens) if lens is not None else None, cmap_dev.data_ptr() if cmap_dev is not None else None,
        cmap.strides[0] if cmap is not None else 0, gu.stream()))
    ref = np.zeros(nvox, np.uint32)
    n_ref, rec, hit = wco.integrate_warped(ref, plain.getDims(), plain.getVoxelSize(), plain.getTruncDist(), plain.getMaxWeight(), depth,
                                           plain.getPose(), world2cam, K, nodes, weight_scale)
    ref_col = np.zeros(nvox, np.uint32)
    n_col_ref = wco.fuse(ref_col, rec, hit, plain.getTruncDist(), plain.getMaxWeight(), img_host, K, cam, lens, cmap)
    torch.cuda.synchronize()
    return (dict(vol=gu.host(plain.data_, np.uint32, -1), act=plain.activity_.cpu().numpy(), counters=c_plain.cpu().numpy()),
            dict(vol=gu.host(coloured.data_, np.uint32, -1), act=coloured.activity_.cpu().numpy(), counters=c_col.cpu().numpy(),
                 colours=gu.host(colours, np.uint32, -1)),
            dict(vol=ref, n=n_ref, colours=ref_col, n_col=n_col_ref))


def _check(plain, col, ref, label, min_col=100):
    assert np.array_equal(plain["vol"], col["vol"]) and np.array_equal(plain["act"], col["act"])
    assert np.array_equal(plain["counters"], col["counters"][:2])
    tsdf_diff = plain["vol"] != ref["vol"]
    col_diff = (col["colours"] != ref["colours"]) & ~tsdf_diff
    n = plain["vol"].size
    print(f"{label}: {int(col['counters'][2])} coloured (oracle {ref['n_col']}), {int(tsdf_diff.sum())} TSDF words differ from the oracle, "
          f"{int(col_diff.sum())} colour words differ elsewhere")
    assert int(tsdf_diff.sum()) <= max(2, int(1e-5 * n))
    assert int(col_diff.sum()) == 0
    assert abs(int(col["counters"][2]) - ref["n_col"]) <= max(2, int(1e-5 * n))
    assert ref["n_col"] >= min_col


CASES = {
    "identity": dict(dim=64, M=300, t=0.0, ws=0.0, pose="identity"),
    "translated_tilted": dict(dim=96, M=500, t=0.002, ws=100.0, pose="tilted"),
    "few_nodes": dict(dim=64, M=40, t=0.01, ws=50.0, pose="tilted"),
}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", list(CASES))
def test_kernel_matches_plain_and_oracle(orc, case, mode):
    c = CASES[case]
    depth = synth.sphere_wall_depth(seed=c["dim"] + c["M"])
    nodes = _surface_nodes(orc, c["M"], seed=c["M"], t_scale=c["t"])
    pose = host.identity_pose() if c["pose"] == "identity" else _tilted_pose()
    _check(*_run_modes(orc, lambda: _volume(c["dim"], 1.0), depth, nodes, pose, c["ws"], mode), f"{case}/{mode}")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("variant", ["rotated", "no_bvh", "no_list", "ragged", "empty"])
def test_kernel_paths_match(orc, monkeypatch, variant, mode):
    dim, M, t, rotate, pose = 64, 200, 0.004, False, _tilted_pose()
    factory = lambda: _volume(dim, 1.0)  # noqa: E731
    depth = synth.sphere_wall_depth(seed=11)
    min_col = 100
    if variant == "rotated":
        rotate = True
    elif variant == "no_bvh":
        dim, M, t, pose = 32, 9000, 0.001, host.identity_pose()
        min_col = 20
    elif variant == "no_list":
        monkeypatch.setenv("DF_FUSION_LIST", "0")
    elif variant == "ragged":
        def factory():
            vol = host.TsdfVolume((40, 28, 36), track_activity=True)
            vol.setTruncDist(0.08); vol.setMaxWeight(MAXW); vol.setSize((1.0, 1.0, 1.0)); vol.setPose(synth.volume_pose(1.0)); vol.clear()
            return vol
        M, t = 150, 0.002
    elif variant == "empty":
        depth = np.zeros_like(depth)
        min_col = 0
    nodes = _surface_nodes(orc, M, seed=5, t_scale=t, rotate=rotate)
    plain, col, ref = _run_modes(orc, factory, depth, nodes, pose, 100.0, mode, pad=3 if variant == "ragged" else 0)
    _check(plain, col, ref, f"{variant}/{mode}", min_col)
    if variant == "empty":
        assert not col["colours"].any() and not col["vol"].any()


@pytest.mark.parametrize("scale", [0.75, 2.0])
def test_colour_image_smaller_and_larger_than_depth(orc, scale):
    depth = synth.sphere_wall_depth(seed=3)
    nodes = _surface_nodes(orc, 300, seed=7, t_scale=0.002)
    _check(*_run_modes(orc, lambda: _volume(64, 1.0), depth, nodes, _tilted_pose(), 100.0, "camera", pad=5, scale=scale), f"scale {scale}")


def test_refusals_write_nothing(orc):
    depth = synth.sphere_wall_depth(seed=3)
    rows, cols = depth.shape
    nodes = _surface_nodes(orc, 100, seed=7)
    wf = host.WarpField()
    wf.setNodes(torch.from_numpy(nodes).cuda())
    vol = _volume(32, 1.0)
    colours = torch.zeros(32 ** 3, dtype=torch.int32, device="cuda")
    img = torch.zeros((rows, cols, 4), dtype=torch.uint8, device="cuda")
    d = host.u16_to_device(depth)
    cam = capi.make_color_camera(K, cols, rows)
    cmap = torch.zeros((rows, cols), dtype=torch.int32, device="cuda")
    bad_lens = capi.Lens()
    bad_lens.r2_max = -1.0
    lib = capi.load()
    I = capi.make_aff(*host.identity_pose())

    def call(depth_pitch=cols * 2, colours_ptr=colours.data_ptr(), bgra=img.data_ptr(), bgra_pitch=cols * 4, cam_=None, lens=None, map_=None,
             map_pitch=0):
        return lib.df_integrate_warped_color(vol._vol(), d.data_ptr(), depth_pitch, cols, rows, capi.make_aff(*vol.pose_), I, capi.make_intr(*K),
                                             wf.nodes_.data_ptr(), len(nodes), wf.grid_.data_ptr(), 0.0, None, vol.activity_.data_ptr(), None,
                                             colours_ptr, bgra, bgra_pitch, cam_, lens, map_, map_pitch, gu.stream())
    before = gu.host(vol.data_, np.uint32, -1).copy()
    inval = 1                                                       # cudaErrorInvalidValue
    for kw in (dict(depth_pitch=cols * 2 - 2), dict(depth_pitch=cols * 2 + 1), dict(colours_ptr=None), dict(bgra=None), dict(bgra_pitch=cols * 4 - 4),
               dict(bgra_pitch=cols * 4 + 2), dict(cam_=C.byref(cam)), dict(cam_=C.byref(cam), map_=cmap.data_ptr(), map_pitch=cols * 4 - 4),
               dict(cam_=C.byref(cam), map_=cmap.data_ptr(), map_pitch=cols * 4, lens=C.byref(bad_lens))):
        assert call(**kw) == inval, kw
    torch.cuda.synchronize()
    assert np.array_equal(gu.host(vol.data_, np.uint32, -1), before) and not colours.any().item()
    assert lib.df_integrate_warped_launch_count() == 4


# ------------------------------------------------------------------------------------------------------------------------ the frame loop
RGBD = [synth.umbrella_rgbd(t) for t in range(8)]
WC = kf.COLOR | kf.WARPED_INTEGRATE | kf.WARPED_COLOR


def _params(flags, dim=128):
    return gu.kinfu_params(dim, flags, max_nodes=1024, cloud_capacity=1_000_000)


@pytest.mark.parametrize("extra", [0, kf.EXTEND_FIELD, kf.LIVE_MODEL], ids=["alone", "extend_field", "live_model"])
def test_colour_never_feeds_back(extra):
    plain, colour = kf.KinFu(_params(kf.WARPED_INTEGRATE | extra)), kf.KinFu(_params(WC | extra))
    for depth, bgra in RGBD[:6]:
        plain(depth)
        colour(depth, bgra)
        assert gu.state(plain) == gu.state(colour)
        for name in ("volume", "nodes", "cloud"):
            assert np.array_equal(plain.buffer(name), colour.buffer(name))
    assert (colour.buffer("color_volume") >> 24).max() == 6
    assert (colour.mesh_colors()[:, 3] == 255).mean() > 0.5
    plain.close(); colour.close()


def _dev_buffer(k, which):
    ptr, pitch, c_, r_ = C.c_void_p(), C.c_size_t(), C.c_int(), C.c_int()
    capi.check(k.lib.df_kinfu_get_buffer(k.h, which, C.byref(ptr), C.byref(pitch), C.byref(c_), C.byref(r_)))
    return ptr.value, pitch.value


def _rebuild_frame(k, colours, bgra, first):
    """what the loop did with this frame's colours, from the public entries: a rigid first frame through df_integrate_color (or
    df_integrate_color_camera_lens with the object's colour camera, lens and occlusion map; the loop's dists), a field frame through
    df_integrate_warped_color on a scratch TSDF volume (the loop's CURR_DEPTH, nodes, pose and, with a camera, its occlusion map)"""
    lib, p = k.lib, k.params
    cam, lens = k.color_camera, k.color_lens
    cam_ref, lens_ref = (None if cam is None else C.byref(cam)), (None if lens is None else C.byref(lens))
    vs = tuple(p.volume_size[i] / p.volume_dims[i] for i in range(3))
    trunc = max(p.tsdf_trunc_dist, np.float32(2.1) * np.float32(max(vs)))
    vol_pose = (np.array(p.volume_pose.R, np.float32).reshape(3, 3), np.array(p.volume_pose.t, np.float32))
    img = gu.dev(bgra)
    ipitch = bgra.shape[1] * 4
    cmap, mpitch = _dev_buffer(k, kf.BUF["color_map"]) if cam is not None else (None, 0)
    pose = k.getCameraPose()
    if first:
        V = capi.make_volume(None, tuple(p.volume_dims), vs, trunc, p.tsdf_max_weight)
        vol2cam = co.aff_mul(co.aff_inv(pose), vol_pose)
        dists, dpitch = _dev_buffer(k, kf.BUF["dists"])
        act, _ = _dev_buffer(k, kf.BUF["activity"])
        if cam is None:
            capi.check(lib.df_integrate_color(V, colours.data_ptr(), dists, dpitch, img.data_ptr(), ipitch, p.cols, p.rows, capi.make_aff(*vol2cam),
                                              p.intr, act, gu.stream()))
        else:
            capi.check(lib.df_integrate_color_camera_lens(V, colours.data_ptr(), dists, dpitch, p.cols, p.rows, capi.make_aff(*vol2cam), p.intr,
                                                          cam, lens_ref, img.data_ptr(), ipitch, cmap, mpitch, act, gu.stream()))
        return
    # the TSDF side is only needed for its voxel walk: a scratch copy of the volume before this frame would be the loop's own, but the
    # colour rule reads only (x_t, pixel, rho), which depend on the frame and the field, not on the volume's contents
    n_vox = int(np.prod(tuple(p.volume_dims)))
    scratch = torch.zeros(n_vox, dtype=torch.int32, device="cuda")
    V = capi.make_volume(scratch.data_ptr(), tuple(p.volume_dims), vs, trunc, p.tsdf_max_weight)
    depth, dpitch = _dev_buffer(k, kf.BUF["curr_depth"])
    nodes, _ = _dev_buffer(k, kf.BUF["nodes"])
    M = k.info()["nodes"]
    grid = torch.empty(int(lib.df_node_grid_bytes(1024)), dtype=torch.uint8, device="cuda")
    capi.check(lib.df_build_node_grid(nodes, M, grid.data_ptr(), gu.stream()))
    capi.check(lib.df_integrate_warped_color(V, depth, dpitch, p.cols, p.rows, p.volume_pose, capi.make_aff(*co.aff_inv(pose)), p.intr, nodes, M,
                                             grid.data_ptr(), p.fusion_weight_scale, None, None, None, colours.data_ptr(), img.data_ptr(), ipitch,
                                             cam_ref, lens_ref, cmap, mpitch, gu.stream()))


# a colour camera of its own beside the depth camera: 960 x 540, 52 mm baseline, a pincushion lens
CAM_K, CAM_COLS, CAM_ROWS = (540.685, 540.685, 479.5, 269.5), 960, 540
CAM_D2C = (np.eye(3, dtype=np.float32), np.array([-0.052, 0.0, 0.0], np.float32))
CAM_LENS = (0.12, 0.03, 0.0005, -0.0004, 0.0)
RGBD_CAM = [synth.umbrella_rgbd(t, color_camera=(CAM_K, CAM_COLS, CAM_ROWS, CAM_D2C, CAM_LENS))[1] for t in range(5)]


@pytest.mark.parametrize("overlap,camera", [("1", False), ("0", False), ("1", True)], ids=["overlap", "no_overlap", "camera_lens"])
def test_loop_colours_rebuilt_from_the_public_entries(monkeypatch, overlap, camera):
    monkeypatch.setenv("DF_KINFU_OVERLAP_EXTRACT", overlap)
    k = kf.KinFu(_params(WC))
    if camera:
        k.set_color_camera(CAM_K, CAM_COLS, CAM_ROWS, CAM_D2C, lens=CAM_LENS)
    mine = torch.zeros(128 ** 3, dtype=torch.int32, device="cuda")
    for t, (depth, bgra) in enumerate(RGBD[:5]):
        image = RGBD_CAM[t] if camera else bgra
        nodes_before = k.info()["nodes"] if t else 0
        k(depth, image)
        _rebuild_frame(k, mine, image, t == 0 or nodes_before < 8)
        torch.cuda.synchronize()
        assert np.array_equal(k.buffer("color_volume"), gu.host(mine, np.uint32, -1)), f"frame {t}"
    assert (k.buffer("color_volume") >> 24).max() == 5
    before = (k.buffer("color_volume").copy(), k.state_digest())
    k(RGBD[5][0])                                                # a depth-only frame: geometry moves on, the colour volume stays
    assert np.array_equal(k.buffer("color_volume"), before[0]) and k.state_digest() != before[1]
    k.close()


def test_host_wrapper_equals_the_c_entry(orc):
    """host.TsdfVolume.integrate_warped_color (pitches from a padded image view and the map tensor, camera and lens by reference) gives what
    the C entry gives on the same inputs"""
    depth = synth.sphere_wall_depth(seed=21)
    rows, cols = depth.shape
    nodes = _surface_nodes(orc, 300, seed=21, t_scale=0.002)
    cam, lens = _camera("camera_lens", cols, rows)
    bgra = np.random.default_rng(21).integers(0, 256, (cam.rows, cam.cols, 4), dtype=np.uint8)
    padded = torch.from_numpy(np.concatenate([bgra, np.zeros((cam.rows, 5, 4), np.uint8)], axis=1)).cuda()
    view = padded[:, :cam.cols]
    cmap = gu.dev(lo.depth_map(depth, K, cam, lens))
    ccam = capi.make_color_camera(cam.K, cam.cols, cam.rows, cam.d2c)
    wf = host.WarpField()
    wf.setNodes(torch.from_numpy(nodes).cuda())
    d = host.u16_to_device(depth)
    a, b = _volume(64, 1.0), _volume(64, 1.0)
    ca, cb = (torch.zeros(64 ** 3, dtype=torch.int32, device="cuda") for _ in range(2))
    na, nb = (torch.zeros(3, dtype=torch.int64, device="cuda") for _ in range(2))
    world2cam = a.integrate_warped_color(d, _tilted_pose(), K, wf, ca, view, 100.0, na, ccam, lens, cmap)
    capi.check(capi.load().df_integrate_warped_color(
        b._vol(), d.data_ptr(), cols * 2, cols, rows, capi.make_aff(*b.pose_), capi.make_aff(*world2cam), capi.make_intr(*K), wf.nodes_.data_ptr(),
        len(nodes), wf.grid_.data_ptr(), 100.0, nb.data_ptr(), b.activity_.data_ptr(), None, cb.data_ptr(), padded.data_ptr(), (cam.cols + 5) * 4,
        C.byref(ccam), C.byref(lens), cmap.data_ptr(), cmap.stride(0) * 4, gu.stream()))
    torch.cuda.synchronize()
    assert int(na[2].item()) > 1000 and torch.equal(na, nb) and torch.equal(ca, cb) and torch.equal(a.data_, b.data_)


def test_snapshot_resume_equals_the_uninterrupted_run(tmp_path):
    a = kf.KinFu(_params(WC))
    for depth, bgra in RGBD[:3]:
        a(depth, bgra)
    path = tmp_path / "wc.snap"
    a.save(path)
    b = kf.KinFu.from_snapshot(path)
    assert b.params.flags & kf.WARPED_COLOR
    for depth, bgra in RGBD[3:6]:
        a(depth, bgra)
        b(depth, bgra)
    assert gu.state(a) == gu.state(b) and np.array_equal(a.buffer("color_volume"), b.buffer("color_volume"))
    a.close(); b.close()


def test_create_refusals_and_environment(capfd, monkeypatch):
    for flags, missing in ((kf.WARPED_INTEGRATE | kf.WARPED_COLOR, "DF_KINFU_COLOR"), (kf.COLOR | kf.WARPED_COLOR, "DF_KINFU_WARPED_INTEGRATE")):
        with pytest.raises(RuntimeError):
            kf.KinFu(_params(flags))
        err = capfd.readouterr().err
        assert "DF_KINFU_WARPED_COLOR" in err and missing in err
    with pytest.raises(RuntimeError):
        kf.KinFu(_params(kf.COLOR | kf.WARPED_INTEGRATE))
    assert "DF_KINFU_WARPED_INTEGRATE" in capfd.readouterr().err
    monkeypatch.setenv("DF_KINFU_WARPED_COLOR", "1")
    k = kf.KinFu(_params(kf.COLOR | kf.WARPED_INTEGRATE))          # the variable completes an object with both flags
    plain = kf.KinFu(_params(kf.WARPED_INTEGRATE))                  # and leaves a colourless one alone
    for depth, bgra in RGBD[:3]:
        k(depth, bgra)
        plain(depth)
    assert gu.state(k) == gu.state(plain) and (k.buffer("color_volume") >> 24).max() == 3
    k.close(); plain.close()


def test_colour_tracking_runs_with_the_flag():
    k = kf.KinFu(_params(WC | kf.COLOR_TRACKING))
    for depth, bgra in RGBD[:5]:
        k(depth, bgra)
    info = k.info()
    assert info["frame_counter"] == 5 and info["nodes"] >= 8
    assert (k.buffer("color_volume") >> 24).max() == 5
    k.close()


# ------------------------------------------------------------------------------------------------------------------------ fidelity
def _cap_score(verts, rgba):
    """(cap vertices, coloured fraction, median and 90th percentile of the per-channel error against the scene's texture) over the cap away
    from its rim, as test_color_gpu.py's fidelity test selects it: canonical coordinates are frame 0's world coordinates"""
    r2 = verts[:, 0] ** 2 + verts[:, 1] ** 2
    cap = (r2 < 0.25 ** 2) & (np.abs(verts[:, 2] - (0.9 + 0.6 * r2)) < 0.05)
    coloured = rgba[:, 3] == 255
    err = np.abs(rgba[cap & coloured][:, :3].astype(int) - synth.umbrella_texture(verts[cap & coloured]).astype(int))
    return int(cap.sum()), float(coloured[cap].mean()), float(np.median(err)) if err.size else 255.0, \
        float(np.percentile(err, 90)) if err.size else 255.0


def test_texture_fidelity_c2_256_through_the_field():
    """20 frames of the deforming umbrella at 256^3 with warped fusion, field extension and DF_KINFU_WARPED_COLOR: the cap's colours match the
    scene's texture.  Negative control: the same frames fused through df_integrate_warped_color with an identity field (each voxel sampled
    where it sits in the canonical volume, not where the surface now is), at the loop's poses, scored at the same vertices: the bars reject it."""
    frames = [synth.umbrella_rgbd(t) for t in range(20)]
    k = kf.KinFu(gu.kinfu_params(256, WC | kf.EXTEND_FIELD, max_nodes=1024, cloud_capacity=2_000_000))
    for depth, bgra in frames:
        k(depth, bgra)
    verts, _, _ = k.mesh()
    verts = np.ascontiguousarray(verts[:, :3], np.float32)
    n_cap, frac, med, p90 = _cap_score(verts, k.mesh_colors())

    p = k.params
    vs = p.volume_size[0] / p.volume_dims[0]
    vol = host.TsdfVolume((256, 256, 256), track_activity=True)
    vol.setSize(tuple(p.volume_size)); vol.setTruncDist(max(p.tsdf_trunc_dist, 2.1 * vs)); vol.setMaxWeight(p.tsdf_max_weight)
    vol.setPose((np.array(p.volume_pose.R, np.float32).reshape(3, 3), np.array(p.volume_pose.t, np.float32)))
    vol.clear()
    nodes = np.ascontiguousarray(k.buffer("nodes").reshape(-1, 12)[:k.info()["nodes"]], np.float32)
    nodes[:, 3:11] = (1, 0, 0, 0, 1, 0, 0, 0)                      # every node the identity DualQuaternion()
    wf = host.WarpField()
    wf.setNodes(torch.from_numpy(nodes).cuda())
    ctrl = torch.zeros(256 ** 3, dtype=torch.int32, device="cuda")
    for t, (depth, bgra) in enumerate(frames):
        vol.integrate_warped_color(host.u16_to_device(depth), k.getCameraPose(t), (p.intr.fx, p.intr.fy, p.intr.cx, p.intr.cy),
                                   wf, ctrl, torch.from_numpy(bgra).cuda(), p.fusion_weight_scale)
    out = torch.zeros(len(verts), dtype=torch.int32, device="cuda")
    pts = torch.from_numpy(verts).cuda()
    capi.check(k.lib.df_sample_colors(vol._vol(), ctrl.data_ptr(), p.volume_pose, 0.5, pts.data_ptr(), 0, 3, len(verts), 1, None, out.data_ptr(), 0,
                                      gu.stream()))
    torch.cuda.synchronize()
    c_cap, c_frac, c_med, c_p90 = _cap_score(verts, out.cpu().numpy().view(np.uint8).reshape(-1, 4))
    k.close()
    line = (f"warped colour: {n_cap} cap vertices, coloured {frac:.4f}, median {med:.1f}, p90 {p90:.1f}; identity field: coloured {c_frac:.4f}, "
            f"median {c_med:.1f}, p90 {c_p90:.1f}")
    print(line)
    out_path = os.environ.get("DF_WARPED_COLOR_FIDELITY_OUT")
    if out_path:
        Path(out_path).write_text(line + "\n")
    # measured (NVIDIA H100 80GB HBM3, 700 W, one run): 28,807 cap vertices; through the field 99.77 % coloured, per-channel error median
    # 20, 90th percentile 48 of 255; the identity field 92.34 % coloured, median 28, p90 64 -- each of its three numbers fails its bar
    assert n_cap > 5000
    passes = lambda f, m, q: f > WC_FIDELITY_MIN_FRACTION and m <= WC_FIDELITY_MEDIAN and q <= WC_FIDELITY_P90  # noqa: E731
    assert passes(frac, med, p90), (frac, med, p90)
    assert not passes(c_frac, c_med, c_p90), (c_frac, c_med, c_p90)


WC_FIDELITY_MIN_FRACTION, WC_FIDELITY_MEDIAN, WC_FIDELITY_P90 = 0.97, 23.0, 56.0     # the measured 0.9977, 20 and 48 with a margin


# ------------------------------------------------------------------------------------------------------------------------ C++ mirror
def test_cpp_mirror_exports_the_same_colours(tmp_path):
    """dfusion_flags 8 | 256 | 1024 through the C++ mirror: the coloured live mesh it writes equals the Python export byte for byte"""
    exe = build.build_cpp_program(ROOT / "tests" / "cpp" / "warped_color_export.cpp", ROOT / "tests" / "cpp" / "_build" / "warped_color_export")
    frames = RGBD[:5]
    np.stack([d for d, _ in frames]).tofile(tmp_path / "depth.u16")
    np.stack([c for _, c in frames]).tofile(tmp_path / "bgra.u8")
    r = subprocess.run([str(exe), str(tmp_path / "depth.u16"), str(tmp_path / "bgra.u8"), str(len(frames)), str(tmp_path / "cpp.ply")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    p = kf.KinFuParams.default_params_dynamicfusion()
    p.flags = WC
    k = kf.KinFu(p)
    for depth, bgra in frames:
        k(depth, bgra)
    assert k.info()["nodes"] >= 8
    k.save_mesh(tmp_path / "py.ply", live=True, colors=True)
    k.close()
    assert (tmp_path / "cpp.ply").read_bytes() == (tmp_path / "py.ply").read_bytes()
