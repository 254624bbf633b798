"""The float64 reference of the TSDF stage (tsdf_reference.py) against the C oracle, on the CPU: the oracle (bit for bit the GPU kernels'
arithmetic) must lie within every bar, with few enough ambiguous voxels and rays that the bars cannot pass by accident, and inputs
perturbed the way a kernel could get them wrong (a half-voxel offset, two voxel sizes swapped, the principal point a pixel off) must land
far outside them."""
import numpy as np
import pytest

import tsdf_cases as tc
import tsdf_reference as tr

pytestmark = pytest.mark.usefixtures("orc")

SMALL = [c for c in tc.VOLUME_CASES if c[0] in ("plain1", "ragged")] + [("v5_aniso", "tilted", tc.DEFAULT_K, "tilted")]
AMB_MAX = 1e-3


def _integrate(orc, name, pose_kind, K, cols=640, rows=480, frames=3):
    """the oracle's volume after each frame: [(prev, after, dists, vol2cam)]"""
    dims = tc.VOLUMES[name][0]
    vs, trunc = tc.voxel_size(name), tc.trunc_dist(name)
    vol = np.zeros(int(np.prod(dims)), np.uint32)
    out = []
    for f in range(frames):
        dists = orc.compute_dists(tc.scene_depth(name, pose_kind, cols, rows, K, f), K)
        v2c = tc.vol2cam(name, pose_kind, f)
        prev = vol.copy()
        orc.integrate(vol, dims, vs, trunc, tc.MAX_W, dists, v2c, K)
        out.append((prev, vol.copy(), dists, v2c))
    return out


def _raycast(orc, name, vol, c2v, K, cols=640, rows=480):
    dims = tc.VOLUMES[name][0]
    Rinv = np.linalg.inv(c2v[0].astype(np.float64)).astype(np.float32)
    rp, rn, _ = orc.raycast_points(vol, dims, tc.voxel_size(name), tc.trunc_dist(name), tc.MAX_W, c2v, Rinv, K, cols, rows,
                                   tc.STEP_FACTOR, tc.DELTA_FACTOR)
    return rp, rn, Rinv


@pytest.mark.parametrize("cols,rows", tc.FRAMES)
def test_dists_round_to_the_float64_ray_length(orc, cols, rows):
    K = tc.frame_K(cols, rows)
    depth = tc.scene_depth("v5_iso", "front", cols, rows, K, 0)
    got = orc.compute_dists(depth, K)
    _, h, amb = tr.dists64(depth, K)
    assert np.array_equal(got[~amb], h[~amb])
    # an ambiguous pixel holds one of the two halves next to the ray length
    near = np.abs(got[amb].view(np.float16).astype(np.float64) - h[amb].view(np.float16).astype(np.float64))
    assert np.all(near <= 2 * tr.halfulp(h[amb].view(np.float16).astype(np.float64)))
    if cols * rows > 1000:
        assert amb.mean() < 1.5e-3, amb.mean()


@pytest.mark.parametrize("case", SMALL, ids=lambda c: f"{c[0]}-{c[1]}")
def test_oracle_lies_within_the_float64_bars(orc, case):
    name, pose_kind, K, view = case
    dims = tc.VOLUMES[name][0]
    vs, trunc = tc.voxel_size(name), tc.trunc_dist(name)
    nvox = int(np.prod(dims))
    for prev, vol, dists, v2c in _integrate(orc, name, pose_kind, K):
        ref = tr.integrate64(prev, dims, vs, trunc, tc.MAX_W, dists, v2c, K)
        bad, ratio, nupd, namb = tr.integrate_check(prev, vol, ref)
        assert bad == 0 and nupd > 10000 and 0.3 < ratio <= 1.0, (bad, ratio, nupd)
        assert namb / nvox < AMB_MAX, namb / nvox
    c2v = tc.cam2vol(name, pose_kind, view)
    rp, rn, Rinv = _raycast(orc, name, vol, c2v, K)
    ref = tr.raycast64(vol, dims, vs, trunc, c2v, Rinv, K, 640, 480, tc.STEP_FACTOR, tc.DELTA_FACTOR)
    bad, rv, rnv, nhit, namb = tr.raycast_check(rp, rn, ref)
    assert bad == 0 and nhit > 1000, (bad, nhit)
    assert namb / ref["pix"].size < AMB_MAX, namb / ref["pix"].size
    pose = tc.f32(tc.volume_pose(name, pose_kind))
    cloud = orc.extract_cloud(vol, dims, vs, trunc, tc.MAX_W, pose, 1 << 20)
    P, B, _, _ = tr.extract64(vol, dims, vs, pose)
    assert len(cloud) == len(P) > 500
    assert np.all(np.abs(cloud[:, :3] - P) <= B)
    Rp = np.linalg.inv(pose[0].astype(np.float64)).astype(np.float32)
    nrm = orc.extract_normals(vol, dims, vs, trunc, tc.MAX_W, cloud, pose, Rp, tc.DELTA_FACTOR)
    N, NB, namb = tr.normals64(vol, dims, vs, cloud, pose, Rp, tc.DELTA_FACTOR)
    assert np.array_equal(np.isnan(nrm[~namb, 0]), np.isnan(N[~namb, 0]))
    m = ~namb & ~np.isnan(N[:, 0])
    assert m.sum() > 0.3 * len(cloud) and np.all(np.abs(nrm[m, :3] - N[m]) <= NB[m])


def _perturbed(name, pose_kind, K, how):
    """(K, voxel size, shift of the volume origin in volume coordinates) with one input changed the way a kernel could get it wrong"""
    vs = tc.voxel_size(name)
    if how == "half_voxel":
        return K, vs, 0.5 * vs
    if how == "swap_vsy_vsz":
        return K, vs[[0, 2, 1]].copy(), np.zeros(3)
    assert how == "cx_plus_1"
    return (K[0], K[1], K[2] + 1.0, K[3]), vs, np.zeros(3)


@pytest.mark.parametrize("how", ["half_voxel", "swap_vsy_vsz", "cx_plus_1"])
def test_perturbed_inputs_land_far_outside_the_bars(orc, how, capsys):
    name, pose_kind, K, view = "ragged", "tilted", tc.K2, "tilted"   # vsy != vsz
    dims = tc.VOLUMES[name][0]
    trunc = tc.trunc_dist(name)
    Kp, vsp, shift = _perturbed(name, pose_kind, K, how)
    prev, vol, dists, v2c = _integrate(orc, name, pose_kind, K, frames=1)[0]
    v2c_p = (v2c[0], (v2c[1] + v2c[0] @ shift.astype(np.float32)).astype(np.float32))
    ref = tr.integrate64(prev, dims, vsp, trunc, tc.MAX_W, dists, v2c_p, Kp)
    bad, ratio, nupd, _ = tr.integrate_check(prev, vol, ref)
    c2v = tc.cam2vol(name, pose_kind, view)
    rp, rn, Rinv = _raycast(orc, name, vol, c2v, K)
    c2v_p = (c2v[0], (c2v[1] + shift).astype(np.float32))
    rref = tr.raycast64(vol, dims, vsp, trunc, c2v_p, Rinv, Kp, 640, 480, tc.STEP_FACTOR, tc.DELTA_FACTOR)
    rbad, rv, rnv, nhit, _ = tr.raycast_check(rp, rn, rref)
    pose = tc.f32(tc.volume_pose(name, pose_kind))
    cloud = orc.extract_cloud(vol, dims, tc.voxel_size(name), trunc, tc.MAX_W, pose, 1 << 20)
    P, B, _, _ = tr.extract64(vol, dims, vsp, (pose[0], (pose[1] + shift).astype(np.float32)))
    eratio = float(np.max(np.abs(cloud[:, :3] - P) / B)) if len(P) == len(cloud) else np.inf
    with capsys.disabled():
        print(f"\n{how}: integrate {bad}/{nupd} voxels outside, worst {ratio:.3g} bars; ray-cast {rbad} outside, worst vertex {rv:.3g} "
              f"normal {rnv:.3g} bars; extraction worst {eratio:.3g} bars")
    assert bad > 0.01 * nupd and ratio > 100
    assert rbad > 100 and max(rv, rnv) > 100
    if how != "cx_plus_1":                        # the intrinsics do not enter the extraction
        assert eratio > 100


def test_kernel_predictor_restates_the_host_rule():
    """integrate_kernel_for: the kernel df_integrate_tracked launches and its z-chunk, for the shapes of tsdf_cases"""
    want = {"v5_iso": (5, 4, 32), "v5_aniso": (5, 4, 32), "v5_deep": (5, 4, 64), "plain4": (0, 4, 32), "plain1": (0, 1, 38), "ragged": (0, 4, 37)}
    for name, (dims, _) in tc.VOLUMES.items():
        args = (tc.DEFAULT_K, tc.vol2cam(name, "front", 0), tc.voxel_size(name), tc.trunc_dist(name), 640, 480, 1280)
        assert tr.integrate_kernel_for(dims, 5, *args) == want[name], name
        assert tr.integrate_kernel_for(dims, 3, *args)[0] == (3 if want[name][0] == 5 else 0)
        assert tr.integrate_kernel_for(dims, 1, *args)[0] == 0
    dims = tc.VOLUMES["v5_iso"][0]
    v2c = tc.vol2cam("v5_iso", "front", 0)
    vs, trunc = tc.voxel_size("v5_iso"), tc.trunc_dist("v5_iso")
    assert tr.integrate_kernel_for(dims, 5, (570.0, 570.0, 0.5, 240.0), v2c, vs, trunc, 640, 480, 1280)[0] == 3      # |cx| < 1
    far = (v2c[0], (v2c[1] + np.float32(70.0)).astype(np.float32))
    assert tr.integrate_kernel_for(dims, 5, tc.DEFAULT_K, far, vs, trunc, 640, 480, 1280)[0] == 3                    # B >= 64 m
    assert tr.integrate_kernel_for(dims, 5, tc.DEFAULT_K, v2c, vs, trunc, 640, 480, 1280, aligned=False) == (0, 1, 32)
