"""GPU parity: TSDF kernels (through the C ABI) vs the CPU oracle on identical seeded inputs.
Bar: bit-exact on the stored u32 voxels and on integer/half images; vertex/normal maps bit-exact too (both sides use the
same IEEE operations in the same order), asserted at 1e-4 relative as the north-star tolerance with the exact-match rate
reported."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from dynamicfusion_b200 import host, synth  # noqa: E402
from kfref_cases import _tilted_pose  # noqa: E402

K = synth.DEFAULT_K


def _setup(dim, size, depth, pose=None):
    vol = host.TsdfVolume((dim, dim, dim))
    vol.setTruncDist(0.04)
    vol.setMaxWeight(64)
    vol.setSize((size, size, size))
    vol.setPose(synth.volume_pose(size))
    vol.setRaycastStepFactor(0.75)
    vol.setGradientDeltaFactor(0.5)
    vol.clear()
    return vol


@pytest.mark.parametrize("dim,pose_kind", [(64, "identity"), (128, "tilted"), (96, "tilted")])
def test_compute_dists_integrate_raycast_match_oracle(orc, dim, pose_kind):
    depth = synth.sphere_wall_depth(seed=dim)
    cam_pose = host.identity_pose() if pose_kind == "identity" else _tilted_pose()
    vol = _setup(dim, 1.0, depth)
    d_depth = host.u16_to_device(depth)

    dists = host.computeDists(d_depth, K)
    dists_ref = orc.compute_dists(depth, K)
    assert np.array_equal(host.u16_from_device(dists), dists_ref)

    # two integrations (weights 1 then 2) from slightly different poses
    ref_vol = np.zeros(dim ** 3, np.uint32)
    n_upd = torch.zeros(1, dtype=torch.int64, device="cuda")
    total_ref = 0
    for pose in (cam_pose, host.aff_mul(cam_pose, (np.eye(3, dtype=np.float32), np.array([0.004, 0.0, 0.002], np.float32)))):
        vol2cam = vol.integrate(dists, pose, K, n_upd)
        total_ref += orc.integrate(ref_vol, vol.getDims(), vol.getVoxelSize(), vol.getTruncDist(), vol.getMaxWeight(), dists_ref, vol2cam, K)
    got = vol.data_.cpu().numpy().view(np.uint32)
    assert int(n_upd.item()) == total_ref
    assert total_ref > 0
    mism = np.count_nonzero(got != ref_vol)
    assert mism == 0, f"{mism} voxels differ out of {dim ** 3}"

    pts, nrm, (cam2vol, Rinv) = vol.raycast(cam_pose, K, 640, 480)
    rp, rn, stats = orc.raycast_points(ref_vol, vol.getDims(), vol.getVoxelSize(), vol.getTruncDist(), vol.getMaxWeight(), cam2vol, Rinv, K,
                                       640, 480, 0.75, 0.5)
    gp, gn = pts.cpu().numpy(), nrm.cpu().numpy()
    assert stats[0] > 1000, "scene produced too few hits to be a meaningful test"
    assert np.array_equal(np.isnan(gp), np.isnan(rp)) and np.array_equal(np.isnan(gn), np.isnan(rn))
    m = ~np.isnan(rp[..., 0])
    np.testing.assert_allclose(gp[m], rp[m], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(gn[m], rn[m], rtol=1e-4, atol=1e-6)
    exact = np.array_equal(gp.view(np.uint32), rp.view(np.uint32)) and np.array_equal(gn.view(np.uint32), rn.view(np.uint32))
    assert exact, "vertex/normal maps are expected to be bit-identical to the oracle"

    # the measurement variant (counters compiled in) must produce the same maps, the oracle's hit count, and a plausible number of
    # unique voxels: no more than the volume holds, nor than every fetched sample plus the 16 + 48 stencil reads of a hit (SURVEY 8d)
    st = vol.raycast_stats(cam_pose, K, 640, 480)
    assert np.array_equal(st["points"].cpu().numpy().view(np.uint32), gp.view(np.uint32))
    assert np.array_equal(st["normals"].cpu().numpy().view(np.uint32), gn.view(np.uint32))
    assert st["hit_rays"] == stats[0]
    assert 1000 < st["unique_voxels"] <= min(dim ** 3, st["march_samples"] + 640 * 480 + 64 * st["hit_rays"])
    assert st["algorithmic_bytes"] == 4 * st["unique_voxels"] + 32 * 640 * 480


def test_clear_volume(orc):
    vol = _setup(32, 1.0, None)
    vol.data_.fill_(-1)
    vol.clear()
    assert int(vol.data_.abs().sum().item()) == 0


def test_integrate_odd_dims_scalar_path(orc):
    """dims not divisible by 4 take the scalar kernel; empty frame (all-zero depth) writes nothing"""
    depth = synth.sphere_wall_depth(seed=3)
    vol = host.TsdfVolume((30, 34, 38))
    vol.setSize((1.0, 1.0, 1.0)); vol.setTruncDist(0.04); vol.setMaxWeight(64); vol.setPose(synth.volume_pose(1.0)); vol.clear()
    dists = host.computeDists(host.u16_to_device(depth), K)
    vol2cam = vol.integrate(dists, host.identity_pose(), K)
    ref = np.zeros(30 * 34 * 38, np.uint32)
    n = orc.integrate(ref, vol.getDims(), vol.getVoxelSize(), vol.getTruncDist(), vol.getMaxWeight(), host.u16_from_device(dists), vol2cam, K)
    assert n > 0 and np.array_equal(vol.data_.cpu().numpy().view(np.uint32), ref)
    vol.clear()
    vol.integrate(torch.zeros_like(dists), host.identity_pose(), K)
    assert int(vol.data_.abs().sum().item()) == 0


def test_max_weight_saturates(orc):
    depth = synth.sphere_wall_depth(seed=1, noise_mm=0.0, dropout=0.0)
    vol = _setup(64, 1.0, depth)
    vol.setMaxWeight(3)
    dists = host.computeDists(host.u16_to_device(depth), K)
    ref = np.zeros(64 ** 3, np.uint32)
    for _ in range(5):
        vol2cam = vol.integrate(dists, host.identity_pose(), K)
        orc.integrate(ref, vol.getDims(), vol.getVoxelSize(), vol.getTruncDist(), 3, host.u16_from_device(dists), vol2cam, K)
    got = vol.data_.cpu().numpy().view(np.uint32)
    assert np.array_equal(got, ref) and (got >> 16).max() == 3


def test_project_and_remove(orc):
    depth = synth.sphere_wall_depth(seed=9)
    rng = np.random.default_rng(2)
    pts = np.full((480, 640, 4), np.nan, np.float32)
    z = rng.uniform(0.5, 1.5, (480, 640)).astype(np.float32)
    u, v = np.meshgrid(np.arange(640, dtype=np.float32), np.arange(480, dtype=np.float32))
    pts[..., 0] = (u + rng.uniform(-40, 40, u.shape).astype(np.float32) - K[2]) / K[0] * z
    pts[..., 1] = (v + rng.uniform(-40, 40, u.shape).astype(np.float32) - K[3]) / K[1] * z
    pts[..., 2] = z
    pts[..., 3] = 0
    pts[rng.random((480, 640)) < 0.3] = np.nan
    d_ref, p_ref = depth.copy(), pts.copy()
    orc.project_and_remove(d_ref, K, p_ref)
    vol = _setup(32, 1.0, None)
    d_dev, p_dev = host.u16_to_device(depth), torch.from_numpy(pts).cuda()
    vol.project_and_remove(d_dev, K, p_dev)
    assert np.array_equal(host.u16_from_device(d_dev), d_ref)
    assert np.array_equal(p_dev.cpu().numpy().view(np.uint32), p_ref.view(np.uint32))
    assert (d_ref == 0).sum() > (depth == 0).sum()


def test_tracked_extraction_equals_full_scan(orc):
    """df_integrate_tracked / df_extract_cloud_tracked: the activity map only lets extraction skip stretches of the volume
    that cannot emit a zero crossing, so points AND their order are those of the full scan (and of the oracle)"""
    dim = 128
    vols = [_setup(dim, 1.0, None), None]
    vols[1] = host.TsdfVolume((dim, dim, dim), track_activity=True)
    v = vols[1]
    v.setTruncDist(0.04); v.setMaxWeight(64); v.setSize((1.0, 1.0, 1.0)); v.setPose(synth.volume_pose(1.0)); v.clear()
    for t in range(3):
        depth = synth.umbrella_depth(t)
        dists = host.computeDists(host.u16_to_device(depth), K)
        pose = synth.camera_drift(4 * t)
        pose = (pose[0].astype(np.float32), pose[1].astype(np.float32))
        for vol in vols:
            vol.integrate(dists, pose, K)
    assert np.array_equal(vols[0].data_.cpu().numpy(), vols[1].data_.cpu().numpy())
    act = vols[1].activity_.cpu().numpy()
    assert 0 < np.count_nonzero(act) < 0.6 * act.size
    clouds = []
    for vol in vols:
        pts, cnt = vol.fetchCloud(600000)
        n = int(cnt.item())
        clouds.append(pts[:n].cpu().numpy())
    assert len(clouds[0]) > 5000
    assert np.array_equal(clouds[0].view(np.uint32), clouds[1].view(np.uint32))
    ref = orc.extract_cloud(vols[0].data_.cpu().numpy().view(np.uint32), vols[0].getDims(), vols[0].getVoxelSize(), vols[0].getTruncDist(),
                            vols[0].getMaxWeight(), vols[0].pose_, 600000)
    assert np.array_equal(clouds[1].view(np.uint32), ref.view(np.uint32))
    # clearing resets the map
    vols[1].clear()
    assert int(vols[1].activity_.sum().item()) == 0 and int(vols[1].fetchCloud(1000)[1].item()) == 0


def _roty(deg, t):
    a = np.deg2rad(deg)
    R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]], np.float32)
    return R, np.asarray(t, np.float32)


@pytest.mark.parametrize("dim", [128, 256])
def test_tracked_raycast_equals_dense_march(orc, dim):
    """df_raycast_points_tracked: the march replays its float chain but only fetches from 8^3 bricks that hold a negative voxel (brick
    table of the activity map).  Maps must be those of the dense march BIT FOR BIT from every viewpoint -- front, oblique, and from
    BEHIND the surface (rays that meet unobserved -> negative -> positive, the (-,+) stop rule) -- and the table must cover exactly
    the bricks that hold negative voxels."""
    v = host.TsdfVolume((dim, dim, dim), track_activity=True)
    v.setTruncDist(0.04); v.setMaxWeight(64); v.setSize((1.0, 1.0, 1.0)); v.setPose(synth.volume_pose(1.0))
    v.setRaycastStepFactor(0.75); v.setGradientDeltaFactor(0.5); v.clear()
    for t in range(3):
        dists = host.computeDists(host.u16_to_device(synth.umbrella_depth(t)), K)
        pose = synth.camera_drift(4 * t)
        v.integrate(dists, (pose[0].astype(np.float32), pose[1].astype(np.float32)), K)
    vol = v.data_.cpu().numpy().view(np.uint32)
    f = (vol & 0xffff).astype(np.uint16).view(np.float16).astype(np.float32).reshape(dim, dim, dim)
    nb = dim // 8
    neg_bricks = (f < 0).reshape(nb, 8, nb, 8, nb, 8).any(axis=(1, 3, 5))
    off = ((dim ** 3 // 1024 + 16) + 255) // 256 * 256
    table = v.activity_.cpu().numpy()[off: off + nb ** 3].reshape(nb, nb, nb) != 0
    # the table is conservative: a voxel that was negative after one integration may have averaged back to >= 0 since
    assert np.all(table[neg_bricks]) and 0 < neg_bricks.mean() < 0.2 and table.sum() <= 1.5 * neg_bricks.sum()
    views = [host.identity_pose(), _tilted_pose(), _roty(30.0, (-0.55, 0.05, 0.25)), _roty(180.0, (0.0, 0.0, 2.3)), _roty(140.0, (0.5, -0.1, 1.9))]
    hits = []
    for cam in views:
        pd, nd, (cam2vol, Rinv) = v.raycast(cam, K, 640, 480, dense=True)
        pt, nt, _ = v.raycast(cam, K, 640, 480)
        assert torch.equal(pd.view(torch.int32), pt.view(torch.int32)) and torch.equal(nd.view(torch.int32), nt.view(torch.int32))
        hits.append(int((~torch.isnan(pd[..., 0])).sum().item()))
    assert hits[0] > 100_000 and min(hits[:3]) > 20_000
    # the dense march against the oracle for the view from behind (the other views are covered by the parity tests above)
    cam = views[3]
    pd, nd, (cam2vol, Rinv) = v.raycast(cam, K, 640, 480)
    rp, rn, _ = orc.raycast_points(vol, v.getDims(), v.getVoxelSize(), v.getTruncDist(), v.getMaxWeight(), cam2vol, Rinv, K, 640, 480, 0.75, 0.5)
    assert np.array_equal(pd.cpu().numpy().view(np.uint32), rp.view(np.uint32)) and np.array_equal(nd.cpu().numpy().view(np.uint32), rn.view(np.uint32))
    # what the skipping buys: unique voxels read by one launch (counting instantiation), front view
    dense = v.raycast_stats(views[0], K, 640, 480, activity_ptr=0)
    tracked = v.raycast_stats(views[0], K, 640, 480)
    assert tracked["hit_rays"] == dense["hit_rays"] == hits[0]
    assert tracked["unique_voxels"] < 0.6 * dense["unique_voxels"]
    print(f"dim {dim}: unique voxels read dense {dense['unique_voxels']} tracked {tracked['unique_voxels']}")


@pytest.mark.parametrize("impl,maxw,frames", [("1", 64, 3), ("3", 64, 3), ("3", 3, 7), ("5", 64, 3), ("5", 3, 7)])
def test_integrate_alternative_kernels_bit_exact_in_subprocess(orc, impl, maxw, frames):
    """the integrate kernel is selected per process (DF_INTEGRATE_IMPL): 1 = plain, 3 = v1 arithmetic + warp-level visibility culling,
    5 (the default) = 3's culling around packed two-voxels-per-instruction arithmetic that replays the IEEE division / square-root fast
    paths; all must store the same u32 voxels as the oracle -- also once the weights saturate (max weight 3, 7 frames); exit code 4 =
    the requested kernel was not the one launched"""
    import os, subprocess, sys
    script = (
        "import numpy as np, torch\n"
        "from dynamicfusion_b200 import host, synth\n"
        "from oracle import orc\n"
        "K = synth.DEFAULT_K; dim = 96\n"
        f"vol = host.TsdfVolume((dim, dim, dim)); vol.setTruncDist(0.04); vol.setMaxWeight({maxw}); vol.setSize((1.0, 1.0, 1.0))\n"
        "vol.setPose(synth.volume_pose(1.0)); vol.clear()\n"
        "ref = np.zeros(dim ** 3, np.uint32)\n"
        f"for t in range({frames}):\n"
        "    depth = synth.umbrella_depth(t)\n"
        "    dists = host.computeDists(host.u16_to_device(depth), K)\n"
        "    R, tr = synth.camera_drift(5 * t); pose = (R.astype(np.float32), tr.astype(np.float32))\n"
        "    vol2cam = vol.integrate(dists, pose, K)\n"
        "    orc.integrate(ref, vol.getDims(), vol.getVoxelSize(), vol.getTruncDist(), vol.getMaxWeight(), orc.compute_dists(depth, K), vol2cam, K)\n"
        "got = vol.data_.cpu().numpy().view(np.uint32)\n"
        "assert np.count_nonzero(ref) > 100000\n"
        "from dynamicfusion_b200 import capi\n"
        f"want = {{'3': 3, '5': 5}}.get('{impl}')\n"
        "if want is not None and capi.load().df_integrate_last_kernel() != want: raise SystemExit(4)\n"
        "raise SystemExit(0 if np.array_equal(got, ref) else 3)\n")
    env = dict(os.environ, DF_INTEGRATE_IMPL=impl)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", script], cwd=root, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.parametrize("case", ["camera_inside", "camera_behind_tilted", "far_volume_falls_back"])
def test_integrate_packed_kernel_domain_edges(orc, case):
    """integrate_kernel_v5 (packed arithmetic) hands runs of voxels next to the camera plane to the scalar slice body and whole launches
    outside its checked domain to v3: the stored voxels must be the oracle's in every case -- a camera inside the volume (voxels behind
    the camera, on its plane, and millimetres in front of it), a tilted camera whose plane cuts the volume obliquely, and intrinsics outside
    the packed kernel's checked domain (df_integrate_last_kernel says which kernel ran)"""
    from dynamicfusion_b200 import capi
    dim = 128
    depth = synth.sphere_wall_depth(seed=7)
    vol = _setup(dim, 1.0, depth)
    Kc = K
    if case == "camera_inside":
        vol.setPose((np.eye(3, dtype=np.float32), np.array([-0.5, -0.5, -0.25], np.float32)))       # camera plane at voxel slice 32
        poses = [host.identity_pose(), (np.eye(3, dtype=np.float32), np.array([0.0, 0.0, 2.0 / dim], np.float32))]   # plane exactly on a slice
        want = 5
    elif case == "camera_behind_tilted":
        vol.setPose((np.eye(3, dtype=np.float32), np.array([-0.5, -0.5, -0.1], np.float32)))
        a = np.deg2rad(25.0)
        R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]], np.float32)
        poses = [(R, np.array([0.02, 0.01, 0.0], np.float32)), _tilted_pose()]
        want = 5
    else:
        # principal point at column 0.5: |cx| < 1 is outside the packed kernel's checked domain (it relies on fma(fx, q, cx) == cx for
        # quotients below 2^-57), so the launch must go to v3
        Kc = (K[0], K[1], 0.5, K[3])
        vol.setPose((np.eye(3, dtype=np.float32), np.array([0.0, -0.5, 0.5], np.float32)))
        poses = [host.identity_pose()]
        want = 3
    vol.clear()
    dists = host.computeDists(host.u16_to_device(depth), Kc)
    dists_ref = orc.compute_dists(depth, Kc)
    ref_vol = np.zeros(dim ** 3, np.uint32)
    n_upd = torch.zeros(1, dtype=torch.int64, device="cuda")
    total = 0
    for pose in poses:
        vol2cam = vol.integrate(dists, pose, Kc, n_upd)
        assert capi.load().df_integrate_last_kernel() == want
        total += orc.integrate(ref_vol, vol.getDims(), vol.getVoxelSize(), vol.getTruncDist(), vol.getMaxWeight(), dists_ref, vol2cam, Kc)
    got = vol.data_.cpu().numpy().view(np.uint32)
    assert total > 10000 and int(n_upd.item()) == total
    mism = np.count_nonzero(got != ref_vol)
    assert mism == 0, f"{case}: {mism} voxels differ"


def test_packed_arithmetic_selftest_on_device():
    """df_integrate_selftest: the packed kernel's division / square-root / running-average sequences against the '/' operator and sqrtf()
    of the same device -- every divisor mantissa at three exponents x 16 dividends (incl. the hard cases a CPU model with a perturbed seed
    fails: all-ones divisor mantissa, power-of-two dividend), every mantissa of the square root's operand at six exponents, 2.7e8 hashed
    pairs over the whole checked domain, every denominator of the running average.  All four counters must be zero."""
    from dynamicfusion_b200 import capi
    mism = torch.full((4,), -1, dtype=torch.int64, device="cuda")
    capi.check(capi.load().df_integrate_selftest(mism.data_ptr(), None))
    torch.cuda.synchronize()
    assert mism.tolist() == [0, 0, 0, 0], mism.tolist()
