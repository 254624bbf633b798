"""Display kernels (df_render_image, df_render_tangent_colors -- what KinFu::renderImage and the reference's demo show) and the
USE_DEPTH-path image operations against the REFERENCE's own kernels (kfusion/src/cuda/imgproc.cu:145-583, tsdf_volume.cu), compiled
for the host into oracle/_ref/libkfref.so.  There is no oracle restatement for these: the comparison is directly with the reference's
code, on inputs the oracle makes on the CPU (the depth ray-cast: on the GPU's own volume, live, where libkfref.so was built).  What the reference's kernels return for those inputs is stored in
tests/golden/render_golden.json (SHA-256 digests) and render_golden.npz (the Phong images), written by tests/golden/make_render_golden.py;
where libkfref.so was built the reference's kernels must still return exactly that.  Bar: tangent colours, depth / normal maps and
ray-cast depth identical; the Phong images within 1 grey level (the reference's __powf / rsqrt are approximate GPU intrinsics)."""
import ctypes as C
import json
from pathlib import Path

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import kfref_cases  # noqa: E402
from dynamicfusion_b200 import capi, host, synth  # noqa: E402
import gpu_util as gu  # noqa: E402

K = synth.DEFAULT_K
LIGHT = (0.3, -0.2, -0.5)
GOLDEN = Path(__file__).parent / "golden"
DIM = 128


def scene(orc):
    """128^3 volume fused from umbrella frame 0 at the identity pose, and its ray-cast maps, by the oracle"""
    dims = np.array([DIM] * 3, np.int32)
    vs = np.full(3, 1.0 / DIM, np.float32)
    vpose, cam = synth.volume_pose(1.0), host.identity_pose()
    vol2cam = host.aff_mul(host.aff_inv(cam), vpose)
    cam2vol = host.aff_mul(host.aff_inv(vpose), cam)
    Rinv = np.linalg.inv(cam2vol[0].astype(np.float64)).astype(np.float32)
    data = np.zeros(DIM ** 3, np.uint32)
    orc.integrate(data, dims, vs, 0.04, 64, orc.compute_dists(synth.umbrella_depth(0), K), vol2cam, K)
    pts, nrm, _ = orc.raycast_points(data, dims, vs, 0.04, 64, cam2vol, Rinv, K, 640, 480, 0.75, 0.5)
    return data, pts, nrm, cam2vol, Rinv


def masked_depth():
    depth = synth.umbrella_depth(2)
    depth[100:140, 200:260] = 0                                              # a hole
    return depth


def reference_outputs(orc):
    """the reference's kernels on the oracle's inputs (needs oracle/_ref/libkfref.so)"""
    ref = orc.load_ref()
    vp = lambda a: C.c_void_p(a.ctypes.data)
    light = (C.c_float * 3)(*LIGHT)
    _, pts, nrm, _, _ = scene(orc)
    out = {}
    rimg, rtan = np.zeros((480, 640, 4), np.uint8), np.zeros((480, 640, 4), np.uint8)
    ref.kfref_render_image(vp(pts), C.c_size_t(640 * 16), vp(nrm), C.c_size_t(640 * 16), 640, 480, orc.intr(*K), light, vp(rimg), C.c_size_t(640 * 4))
    ref.kfref_render_tangent_colors(vp(nrm), C.c_size_t(640 * 16), 640, 480, vp(rtan), C.c_size_t(640 * 4))
    out["render_image"], out["tangent_colors"] = rimg, np.where(~np.isnan(nrm[..., :1]), rtan, 0).astype(np.uint8)
    d_ref, n_ref = masked_depth(), np.zeros((480, 640, 4), np.float32)
    ref.kfref_normals_mask_depth(orc.intr(*K), vp(d_ref), C.c_size_t(640 * 2), 640, 480, vp(n_ref), C.c_size_t(640 * 16))
    out["masked_depth"], out["depth_normals"] = d_ref, n_ref
    dd_ref, nd_ref = np.zeros((240, 320), np.uint16), np.zeros((240, 320, 4), np.float32)
    ref.kfref_resize_depth_normals(vp(d_ref), C.c_size_t(640 * 2), vp(n_ref), C.c_size_t(640 * 16), 640, 480, vp(dd_ref), C.c_size_t(320 * 2), vp(nd_ref),
                                   C.c_size_t(320 * 16))
    out["resized_depth"], out["resized_normals"] = dd_ref, nd_ref
    rimg_d = np.zeros((480, 640, 4), np.uint8)
    ref.kfref_render_image_depth(vp(d_ref), C.c_size_t(640 * 2), vp(n_ref), C.c_size_t(640 * 16), 640, 480, orc.intr(*K), light, vp(rimg_d), C.c_size_t(640 * 4))
    out["render_image_depth"] = rimg_d
    c2d = np.zeros((480, 640), np.uint16)
    ref.kfref_cloud_to_depth(vp(pts), C.c_size_t(640 * 16), 640, 480, vp(c2d), C.c_size_t(640 * 2))
    out["cloud_to_depth"] = np.where(~np.isnan(pts[..., 2]), c2d, 0).astype(np.uint16)
    return out


IMAGES = ("render_image", "render_image_depth")


@pytest.fixture(scope="module")
def golden(orc):
    digests = json.loads((GOLDEN / "render_golden.json").read_text())
    with np.load(GOLDEN / "render_golden.npz") as z:
        images = {k: z[k] for k in IMAGES}
    if orc.reference_available():                                            # the stored outputs are still the reference's
        live = reference_outputs(orc)
        assert {k: kfref_cases.digest(v) for k, v in live.items() if k not in IMAGES} == digests
        assert all(np.array_equal(live[k], images[k]) for k in IMAGES)
    return digests, images


def test_render_kernels_match_the_reference_code(orc, golden):
    digests, images = golden
    _, pts, nrm, _, _ = scene(orc)
    assert np.count_nonzero(~np.isnan(pts[..., 0])) > 100_000
    light = (C.c_float * 3)(*LIGHT)
    lib = capi.load()
    p_dev, n_dev = gu.dev(pts), gu.dev(nrm)
    img = torch.zeros((480, 640, 4), dtype=torch.uint8, device="cuda")
    tan = torch.zeros_like(img)
    capi.check(lib.df_render_image(p_dev.data_ptr(), 640 * 16, n_dev.data_ptr(), 640 * 16, 640, 480, light, img.data_ptr(), 640 * 4, None))
    capi.check(lib.df_render_tangent_colors(n_dev.data_ptr(), 640 * 16, 640, 480, tan.data_ptr(), 640 * 4, None))
    torch.cuda.synchronize()
    gi, gt = img.cpu().numpy(), tan.cpu().numpy()
    rimg = images["render_image"]
    assert np.abs(gi.astype(np.int16) - rimg.astype(np.int16)).max() <= 1
    assert np.mean(gi != rimg) < 0.02
    valid = ~np.isnan(nrm[..., 0])
    assert kfref_cases.digest(np.where(valid[..., None], gt, 0).astype(np.uint8)) == digests["tangent_colors"]
    assert len(np.unique(gi[valid][:, 0])) > 50 and len(np.unique(gi[~valid][:, 0])) > 50      # a shaded surface over the gradient background


def test_depth_path_image_ops_match_the_reference_code(orc, golden):
    """cuda/imgproc.hpp functions of the reference's USE_DEPTH path (computeNormalsAndMaskDepth, resizeDepthNormals, cloudToDepth,
    renderImage(depth)) and the depth variant of the ray-cast: bit-exact against the reference's own kernels (Phong image: 1 level)"""
    digests, images = golden
    lib = capi.load()
    depth = masked_depth()
    # computeNormalsAndMaskDepth
    d_dev = host.u16_to_device(depth)
    n_dev = torch.zeros((480, 640, 4), dtype=torch.float32, device="cuda")
    capi.check(lib.df_normals_mask_depth(capi.make_intr(*K), d_dev.data_ptr(), 640 * 2, 640, 480, n_dev.data_ptr(), 640 * 16, None))
    gd, gn = host.u16_from_device(d_dev), n_dev.cpu().numpy()
    assert kfref_cases.digest(gd) == digests["masked_depth"] and np.count_nonzero(gd != depth) > 500
    assert kfref_cases.digest(gn) == digests["depth_normals"]
    # resizeDepthNormals
    dd = torch.zeros((240, 320), dtype=torch.int16, device="cuda")
    nd = torch.zeros((240, 320, 4), dtype=torch.float32, device="cuda")
    capi.check(lib.df_resize_depth_normals(d_dev.data_ptr(), 640 * 2, n_dev.data_ptr(), 640 * 16, 640, 480, dd.data_ptr(), 320 * 2, nd.data_ptr(), 320 * 16, None))
    assert kfref_cases.digest(host.u16_from_device(dd)) == digests["resized_depth"]
    assert kfref_cases.digest(nd.cpu().numpy()) == digests["resized_normals"]
    # renderImage(depth)
    light = (C.c_float * 3)(*LIGHT)
    img = torch.zeros((480, 640, 4), dtype=torch.uint8, device="cuda")
    capi.check(lib.df_render_image_depth(d_dev.data_ptr(), 640 * 2, n_dev.data_ptr(), 640 * 16, 640, 480, capi.make_intr(*K), light, img.data_ptr(), 640 * 4, None))
    gi, rimg = img.cpu().numpy(), images["render_image_depth"]
    assert np.abs(gi.astype(np.int16) - rimg.astype(np.int16)).max() <= 1 and np.mean(gi != rimg) < 0.02
    # cloudToDepth on the oracle's ray-cast points
    _, pts, _, _, _ = scene(orc)
    rc = torch.zeros((480, 640), dtype=torch.int16, device="cuda")
    p_dev = gu.dev(pts)
    capi.check(lib.df_cloud_to_depth(p_dev.data_ptr(), 640 * 16, 640, 480, rc.data_ptr(), 640 * 2, None))
    assert kfref_cases.digest(host.u16_from_device(rc)) == digests["cloud_to_depth"]
    # ray-cast, depth variant = the points variant of the GPU + cloudToDepth, against the reference's raycast(depth) on the same
    # GPU-fused volume: the reference's kernel runs live, so this part needs its host build
    if not orc.reference_available():
        return
    ref = orc.load_ref()
    vp = lambda a: C.c_void_p(a.ctypes.data)
    vol = host.TsdfVolume((DIM, DIM, DIM))
    vol.setTruncDist(0.04); vol.setMaxWeight(64); vol.setSize((1.0, 1.0, 1.0)); vol.setPose(synth.volume_pose(1.0))
    vol.setRaycastStepFactor(0.75); vol.setGradientDeltaFactor(0.5); vol.clear()
    pose = host.identity_pose()
    vol.integrate(host.computeDists(host.u16_to_device(synth.umbrella_depth(0)), K), pose, K)
    gpts, _, (cam2vol, Rinv) = vol.raycast(pose, K, 640, 480)
    capi.check(lib.df_cloud_to_depth(gpts.data_ptr(), 640 * 16, 640, 480, rc.data_ptr(), 640 * 2, None))
    g_rc = host.u16_from_device(rc)
    volume = vol.data_.cpu().numpy().view(np.uint32)
    rd, rn = np.zeros((480, 640), np.uint16), np.zeros((480, 640, 4), np.float32)
    ref.kfref_raycast_depth(orc.volume(volume, vol.getDims(), vol.getVoxelSize(), vol.getTruncDist(), vol.getMaxWeight()), orc.aff(*cam2vol), orc._f9(Rinv),
                            orc.intr(*K), 640, 480, C.c_float(0.75), C.c_float(0.5), vp(rd), C.c_size_t(640 * 2), vp(rn), C.c_size_t(640 * 16))
    assert np.array_equal(g_rc, rd) and np.count_nonzero(rd) > 100_000
