"""GPU parity at BASELINE.json's other configurations (the bench line is C2; these are parity cases, not bench lines):
C1 256^3 rigid-only single frame, C3 512^3 with 4k warp nodes and 5 LM iterations, C4 768^3 with 1280x720 depth.
Direct oracle comparisons where the oracle finishes in seconds, plus size-independent properties at full size."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from dynamicfusion_b200 import host, kinfu as kf, synth  # noqa: E402
import gpu_util as gu  # noqa: E402

K = synth.DEFAULT_K


def test_c1_256_rigid_single_frame(orc):
    """configs[0]: one 640x480 frame into a 256^3 volume, rigid-only integrate + ray-cast: bit-exact (no expf on this path)"""
    from oracle import orc_pipe
    p = gu.kinfu_params(256, kf.RIGID_ONLY, max_nodes=2048, cloud_capacity=4_000_000, K=K, cols=640, rows=480)
    gpu, cpu = kf.KinFu(p), orc_pipe.KinFu(orc_pipe.params_from(p))
    d = synth.sphere_wall_depth(seed=11)
    assert gpu(d) is False and cpu(d) is False
    assert np.array_equal(gpu.buffer("volume"), cpu.buffer("volume"))
    # second frame: ICP + integrate + ray-cast of the new pose
    d1 = synth.sphere_wall_depth(seed=12)
    assert gpu(d1) is True and cpu(d1) is True
    Rg, tg = gpu.getCameraPose(1)
    Rc, tc = cpu.getCameraPose(1)
    assert np.abs(Rg - Rc).max() < 2e-4 and np.abs(tg - tc).max() < 2e-4
    fg, wg = gu.tsdf(gpu.buffer("volume"))
    fc, wc = gu.tsdf(cpu.buffer("volume"))
    assert np.mean(wg != wc) < 2e-3
    same = wg == wc
    assert np.mean(np.abs(fg[same] - fc[same]) > 2e-3) < 2e-3
    pg, pc = gpu.buffer("prev_points"), cpu.buffer("prev_points")
    both = ~np.isnan(pg[..., 0]) & ~np.isnan(pc[..., 0])
    assert both.sum() > 100_000 and np.mean(np.isnan(pg[..., 0]) != np.isnan(pc[..., 0])) < 5e-3
    assert np.median(np.abs(pg[both][:, :3] - pc[both][:, :3])) < 1e-4
    gpu.close(); cpu.close()


def test_c3_512_4k_nodes_five_lm_iterations(orc):
    """configs[2]: 512^3, 4k warp nodes, k = 8 DQB, 5 LM iterations per frame -- three frames against the oracle's loop"""
    from oracle import orc_pipe
    p = gu.kinfu_params(512, 0, max_nodes=4096, cloud_capacity=4_000_000, K=K, cols=640, rows=480)
    p.solver_nonlinear_iters = 5
    gpu, cpu = kf.KinFu(p), orc_pipe.KinFu(orc_pipe.params_from(p))
    for t in range(3):
        d = synth.umbrella_depth(t)
        assert gpu(d) == cpu(d) == (t > 0)
    gi, ci = gpu.info(), cpu.info()
    assert gi["nodes"] == ci["nodes"] and 3500 <= gi["nodes"] <= 4096
    for t in range(3):
        Rg, tg = gpu.getCameraPose(t)
        Rc, tc = cpu.getCameraPose(t)
        assert np.abs(Rg - Rc).max() < 2e-4 and np.abs(tg - tc).max() < 2e-4, t
    ng, nc = gpu.buffer("nodes")[: gi["nodes"]], cpu.buffer("nodes")
    assert np.array_equal(ng[:, :7], nc[:, :7])
    tg, tc = 2 * ng[:, 8:11], 2 * nc[:, 8:11]
    scale = max(np.abs(tc).max(), 1e-6)
    assert np.median(np.abs(tg - tc)) <= 5e-3 * scale + 2e-6
    sg, sc = gpu.buffer("solve_stats"), cpu.buffer("solve_stats")
    assert abs(sg[3] - sc[3]) <= 0.01 * sc[3] and abs(sg[1] - sc[1]) <= 5e-2 * sc[1]
    fg, wg = gu.tsdf(gpu.buffer("volume"))
    fc, wc = gu.tsdf(cpu.buffer("volume"))
    assert np.mean(wg != wc) < 2e-2
    gpu.close(); cpu.close()


def test_c4_768_hd_depth_integrate_raycast(orc):
    """configs[3]: 768^3 volume, 1280x720 depth -- dists, two integrations and the ray-cast are bit-exact vs the oracle;
    re-integrating the same frame is idempotent on the tsdf and only bumps the weight (size-independent property)"""
    cols, rows = 1280, 720
    K_hd = (K[0] * 2, K[1] * 2, K[2] * 2 + 0.5, K[3] * 1.5 + 0.25)
    depth = synth.umbrella_depth(0, cols=cols, rows=rows, K=K_hd, drift=False)
    dim = 768
    vol = host.TsdfVolume((dim, dim, dim))
    vol.setTruncDist(0.04); vol.setMaxWeight(64); vol.setSize((1.0, 1.0, 1.0)); vol.setPose(synth.volume_pose(1.0))
    vol.setRaycastStepFactor(0.75); vol.setGradientDeltaFactor(0.5); vol.clear()
    d_dev = host.u16_to_device(depth)
    dists = host.computeDists(d_dev, K_hd)
    dists_ref = orc.compute_dists(depth, K_hd)
    assert np.array_equal(host.u16_from_device(dists), dists_ref)
    pose = host.identity_pose()
    n_upd = torch.zeros(1, dtype=torch.int64, device="cuda")
    vol2cam = vol.integrate(dists, pose, K_hd, n_upd)
    first = vol.data_.clone()
    n1 = int(n_upd.item())
    assert n1 > 50_000_000
    ref = np.zeros(dim ** 3, np.uint32)
    n_ref = orc.integrate(ref, vol.getDims(), vol.getVoxelSize(), vol.getTruncDist(), vol.getMaxWeight(), dists_ref, vol2cam, K_hd)
    assert n1 == n_ref
    got = first.cpu().numpy().view(np.uint32)
    assert np.count_nonzero(got != ref) == 0
    # idempotence: same frame, same pose -> (t*1 + t)/2 == t, weight 1 -> 2
    vol.integrate(dists, pose, K_hd, n_upd)
    again = vol.data_.cpu().numpy().view(np.uint32)
    touched = (got >> 16) == 1
    assert int(n_upd.item()) == 2 * n1 and touched.sum() == n1
    assert np.array_equal(again[touched] & 0xffff, got[touched] & 0xffff) and np.all((again[touched] >> 16) == 2)
    assert np.array_equal(again[~touched], got[~touched])
    del got, again, touched, first
    pts, nrm, (cam2vol, Rinv) = vol.raycast(pose, K_hd, cols, rows)
    orc.integrate(ref, vol.getDims(), vol.getVoxelSize(), vol.getTruncDist(), vol.getMaxWeight(), dists_ref, vol2cam, K_hd)
    rp, rn, stats = orc.raycast_points(ref, vol.getDims(), vol.getVoxelSize(), vol.getTruncDist(), vol.getMaxWeight(), cam2vol, Rinv, K_hd, cols, rows, 0.75, 0.5)
    gp, gn = pts.cpu().numpy(), nrm.cpu().numpy()
    assert stats[0] > 300_000
    assert np.array_equal(np.isnan(gp), np.isnan(rp))
    m = ~np.isnan(rp[..., 0])
    np.testing.assert_allclose(gp[m], rp[m], rtol=1e-4, atol=1e-6)
    assert np.array_equal(gp.view(np.uint32), rp.view(np.uint32)) and np.array_equal(gn.view(np.uint32), rn.view(np.uint32))


def test_c4_768_hd_full_loop_two_frames(orc):
    """configs[3] through the whole frame loop (the largest sizes the path is specified for): 768^3 / 1.5 m volume, 1280x720 depth,
    two frames against the oracle's loop -- first frame bit-exact, second frame (ICP + warp + solve + fusion) statistically"""
    from oracle import orc_pipe
    cols, rows = 1280, 720
    K_hd = (K[0] * 2, K[1] * 2, 640.0, 360.0)
    p = gu.kinfu_params(768, 0, max_nodes=2048, cloud_capacity=4_000_000, K=K_hd, cols=cols, rows=rows)
    for i in range(3):
        p.volume_size[i] = 1.5
    p.volume_pose.t[0] = -0.75; p.volume_pose.t[1] = -0.75; p.volume_pose.t[2] = 0.5
    gpu, cpu = kf.KinFu(p), orc_pipe.KinFu(orc_pipe.params_from(p))
    d0 = synth.umbrella_depth(0, cols=cols, rows=rows, K=K_hd)
    assert gpu(d0) is False and cpu(d0) is False
    assert np.array_equal(gpu.buffer("volume"), cpu.buffer("volume"))
    gi, ci = gpu.info(), cpu.info()
    assert gi["nodes"] == ci["nodes"] >= 1000 and gi["cloud_points"] == ci["cloud_points"] > 200_000
    d1 = synth.umbrella_depth(1, cols=cols, rows=rows, K=K_hd)
    assert gpu(d1) is True and cpu(d1) is True
    Rg, tg = gpu.getCameraPose(1)
    Rc, tc = cpu.getCameraPose(1)
    assert np.abs(Rg - Rc).max() < 2e-4 and np.abs(tg - tc).max() < 2e-4
    fg, wg = gu.tsdf(gpu.buffer("volume"))
    fc, wc = gu.tsdf(cpu.buffer("volume"))
    assert np.mean(wg != wc) < 2e-2
    sg, sc = gpu.buffer("solve_stats"), cpu.buffer("solve_stats")
    assert abs(sg[3] - sc[3]) <= 0.01 * sc[3] and abs(sg[1] - sc[1]) <= 5e-2 * sc[1]
    gpu.close(); cpu.close()
