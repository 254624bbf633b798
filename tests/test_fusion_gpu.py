"""GPU parity: per-voxel warped integration (df_integrate_warped, csrc/fusion.cu) vs the CPU oracle (oracle/orc_fusion.c) on identical
seeded inputs, through the C ABI.  Bar: the stored u32 voxels are compared bit for bit.  The only operation on this path that is not
the same IEEE operation on both sides is the double-precision exp() of the node weights (CUDA libm vs glibc, both < 1 ulp and then
narrowed to float); a difference there can flip a gate for a voxel sitting exactly on it, so the tests allow a 1e-5 fraction of
differing voxels and print the count (0 in every run so far)."""
import ctypes as C
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from dynamicfusion_b200 import host, synth  # noqa: E402
from warp_cases import K, MAXW, _surface_nodes, _tilted_pose, _volume  # noqa: E402


def _run_both(orc, dim, size, nodes, depth, cam_pose, weight_scale, passes=2):
    vol = _volume(dim, size)
    wf = host.WarpField()
    wf.setNodes(torch.from_numpy(nodes).cuda())
    d_depth = host.u16_to_device(depth)
    counters = torch.zeros(2, dtype=torch.int64, device="cuda")
    ref = np.zeros(dim ** 3, np.uint32)
    n_ref = 0
    for i in range(passes):
        pose = cam_pose if i == 0 else host.aff_mul(cam_pose, (np.eye(3, dtype=np.float32), np.array([0.003, 0.0, 0.002], np.float32)))
        world2cam = vol.integrate_warped(d_depth, pose, K, wf, weight_scale, counters)
        n_ref += orc.integrate_warped(ref, vol.getDims(), vol.getVoxelSize(), vol.getTruncDist(), vol.getMaxWeight(), depth, vol.getPose(),
                                      world2cam, K, nodes, weight_scale)
    torch.cuda.synchronize()
    got = vol.data_.cpu().numpy().view(np.uint32)
    c = counters.cpu().numpy()
    return vol, got, ref, int(c[0]), int(c[1]), n_ref


def _assert_parity(got, ref, n_got, n_ref, dim):
    mism = int(np.count_nonzero(got != ref))
    print(f"warped integrate {dim}^3: {n_got} voxels written (oracle {n_ref}), {mism} differ")
    assert n_ref > 1000, "scene writes too few voxels to be a meaningful test"
    assert mism <= max(2, int(1e-5 * dim ** 3)), f"{mism} voxels differ out of {dim ** 3}"
    assert abs(n_got - n_ref) <= max(2, int(1e-5 * dim ** 3))


@pytest.mark.parametrize("dim,M,t_scale,weight_scale,pose_kind", [
    (64, 300, 0.0, 0.0, "identity"),          # identity field, unit weights
    (96, 500, 0.002, 100.0, "tilted"),        # small translations: the displacement bound is ~1.6 cm, culling active
    (64, 40, 0.01, 50.0, "tilted"),           # M < 64: the oracle's exhaustive k-NN path; large displacement bound
    (128, 2000, 0.001, 100.0, "identity"),    # node count of the bench configuration
])
def test_integrate_warped_matches_oracle(orc, dim, M, t_scale, weight_scale, pose_kind):
    depth = synth.sphere_wall_depth(seed=dim + M)
    nodes = _surface_nodes(orc, M, seed=M, t_scale=t_scale)
    cam = host.identity_pose() if pose_kind == "identity" else _tilted_pose()
    vol, got, ref, n_got, n_warped, n_ref = _run_both(orc, dim, 1.0, nodes, depth, cam, weight_scale)
    _assert_parity(got, ref, n_got, n_ref, dim)
    assert n_got <= n_warped <= 2 * dim ** 3
    # the activity map must cover every voxel that can emit a zero crossing (W != 0 and F != 1), as df_integrate_tracked guarantees
    act = vol.activity_.cpu().numpy()
    active_vox = np.flatnonzero(((got >> 16) != 0) & ((got & 0xffff) != 0x3c00))
    assert np.all(act[active_vox // 1024] == 1)


def test_integrate_warped_ragged_dims_and_empty_frame(orc):
    """dims that are not multiples of the 32 x 8 block footprint (edge warps carry idle lanes through the warp-wide visibility test),
    anisotropic voxels; an all-zero depth frame writes nothing"""
    dims, size = (40, 28, 36), 1.0
    depth = synth.sphere_wall_depth(seed=4)
    nodes = _surface_nodes(orc, 150, seed=3, t_scale=0.002)
    vol = host.TsdfVolume(dims, track_activity=True)
    vol.setTruncDist(0.08); vol.setMaxWeight(MAXW); vol.setSize((size, size, size)); vol.setPose(synth.volume_pose(size)); vol.clear()
    wf = host.WarpField()
    wf.setNodes(torch.from_numpy(nodes).cuda())
    counters = torch.zeros(2, dtype=torch.int64, device="cuda")
    vol.integrate_warped(host.u16_to_device(np.zeros_like(depth)), _tilted_pose(), K, wf, 100.0, counters)
    torch.cuda.synchronize()
    assert int(counters[0].item()) == 0 and int(vol.data_.abs().sum().item()) == 0
    counters.zero_()
    world2cam = vol.integrate_warped(host.u16_to_device(depth), _tilted_pose(), K, wf, 100.0, counters)
    ref = np.zeros(dims[0] * dims[1] * dims[2], np.uint32)
    n_ref = orc.integrate_warped(ref, vol.getDims(), vol.getVoxelSize(), vol.getTruncDist(), vol.getMaxWeight(), depth, vol.getPose(), world2cam, K,
                                 nodes, 100.0)
    torch.cuda.synchronize()
    got = vol.data_.cpu().numpy().view(np.uint32)
    mism = int(np.count_nonzero(got != ref))
    print(f"ragged {dims}: {int(counters[0].item())} written (oracle {n_ref}), {mism} differ")
    assert n_ref > 500 and mism <= 2 and abs(int(counters[0].item()) - n_ref) <= 2


def test_integrate_warped_rotated_nodes_disable_culling_and_still_match(orc):
    """any rotated node makes the displacement bound infinite: every voxel is warped, the result still equals the oracle's"""
    dim = 64
    depth = synth.sphere_wall_depth(seed=11)
    nodes = _surface_nodes(orc, 200, seed=5, t_scale=0.004, rotate=True)
    _, got, ref, n_got, n_warped, n_ref = _run_both(orc, dim, 1.0, nodes, depth, _tilted_pose(), 100.0, passes=1)
    _assert_parity(got, ref, n_got, n_ref, dim)
    assert n_warped == dim ** 3


def test_integrate_warped_without_bvh_uses_the_grid_walk(orc):
    """more than 8192 nodes: the node grid carries no BVH, every voxel takes knn8_grid -- same answer"""
    dim = 32
    depth = synth.sphere_wall_depth(seed=2)
    nodes = _surface_nodes(orc, 9000, seed=9, t_scale=0.001)
    _, got, ref, n_got, _, n_ref = _run_both(orc, dim, 1.0, nodes, depth, host.identity_pose(), 100.0, passes=1)
    _assert_parity(got, ref, n_got, n_ref, dim)


def test_full_size_weight_conservation(orc):
    """size-independent property at the bench volume (512^3, ~2 k nodes, 640x480): with unit sample weights every written voxel
    gains exactly one unit of weight per pass, so the volume's total weight equals the kernel's own count of written voxels, and a
    second identical pass writes the same voxels again"""
    dim = 512
    depth = synth.umbrella_depth(3)
    nodes = _surface_nodes(orc, 2000, seed=1, t_scale=0.0015)
    wf = host.WarpField()
    wf.setNodes(torch.from_numpy(nodes).cuda())
    d_depth = host.u16_to_device(depth)
    vol = _volume(dim, 1.0)
    counters = torch.zeros(2, dtype=torch.int64, device="cuda")
    vol.integrate_warped(d_depth, _tilted_pose(), K, wf, 0.0, counters)
    torch.cuda.synchronize()
    n1 = int(counters[0].item())
    w = (vol.data_ >> 16) & 0xffff
    assert n1 > 1_000_000 and int(w.sum().item()) == n1 and int(w.max().item()) == 1
    vol.integrate_warped(d_depth, _tilted_pose(), K, wf, 0.0, counters)
    torch.cuda.synchronize()
    w = (vol.data_ >> 16) & 0xffff
    assert int(counters[0].item()) == 2 * n1 and int(w.sum().item()) == 2 * n1 and int((w == 1).sum().item()) == 0
    print(f"512^3: {n1} voxels written per pass, {int(counters[1].item()) // 2} warped")


def test_culling_is_invisible(orc):
    """the visibility culling may only skip voxels that would not have been written: culled and unculled runs (256^3, ~2 k nodes) store
    identical volumes and write the same number of voxels"""
    dim = 256
    depth = synth.umbrella_depth(3)
    nodes = _surface_nodes(orc, 2000, seed=1, t_scale=0.0015)
    nodes[:, 2] = np.where(nodes[:, 2] > 1.2, 1.3, nodes[:, 2])
    wf = host.WarpField()
    wf.setNodes(torch.from_numpy(nodes).cuda())
    d_depth = host.u16_to_device(depth)
    out = []
    for cull in ("1", "0"):
        os.environ["DF_FUSION_CULL"] = cull
        try:
            vol = _volume(dim, 1.0)
            counters = torch.zeros(2, dtype=torch.int64, device="cuda")
            vol.integrate_warped(d_depth, _tilted_pose(), K, wf, 100.0, counters)
            torch.cuda.synchronize()
            out.append((vol.data_.clone(), counters.cpu().numpy().copy()))
            del vol
        finally:
            os.environ.pop("DF_FUSION_CULL", None)
    (va, ca), (vb, cb) = out
    assert int(ca[0]) == int(cb[0]) and int(ca[0]) > 100_000
    assert int(cb[1]) == dim ** 3 and int(ca[1]) < int(cb[1])
    assert torch.equal(va, vb)
    print(f"256^3: {int(ca[0])} voxels written; warped {int(ca[1])} with culling vs {int(cb[1])} without")


def test_candidate_lists_equal_the_tree_search(orc):
    """round 2: per-run candidate lists (DF_FUSION_LIST, default on) must find exactly the neighbours the per-voxel branch-and-bound finds, and
    their local displacement bound may only skip voxels that would not have been written -- 256^3, ~2 k nodes, a handful of 'rim' nodes
    carrying decimetre translations so that the global bound (8 max |t| = metres) culls nothing, as in the live loop"""
    dim = 256
    depth = synth.umbrella_depth(3)
    nodes = _surface_nodes(orc, 2000, seed=1, t_scale=0.0015)
    lib = orc.load()
    for i in (5, 700, 1500):
        lib.orc_node_encode_translation(C.c_void_p(nodes[i].ctypes.data), C.c_float(0.3), C.c_float(-0.2), C.c_float(0.25))
    wf = host.WarpField()
    wf.setNodes(torch.from_numpy(nodes).cuda())
    d_depth = host.u16_to_device(depth)
    out = []
    for use_list in ("1", "0"):
        os.environ["DF_FUSION_LIST"] = use_list
        try:
            vol = _volume(dim, 1.0)
            counters = torch.zeros(2, dtype=torch.int64, device="cuda")
            for _ in range(2):
                vol.integrate_warped(d_depth, _tilted_pose(), K, wf, 100.0, counters)
            torch.cuda.synchronize()
            out.append((vol.data_.clone(), vol.activity_.clone(), counters.cpu().numpy().copy()))
            del vol
        finally:
            os.environ.pop("DF_FUSION_LIST", None)
    (va, aa, ca), (vb, ab, cb) = out
    assert int(ca[0]) == int(cb[0]) and int(ca[0]) > 100_000
    assert torch.equal(va, vb) and torch.equal(aa, ab)
    assert int(cb[1]) == 2 * dim ** 3, "the global bound was expected to cull nothing here"
    assert int(ca[1]) < int(cb[1])
    print(f"256^3: {int(ca[0])} voxels written; warped {int(ca[1])} with candidate lists (local bound) vs {int(cb[1])} with the global bound")


def test_pipeline_with_warped_integration_tracks_the_oracle_pipeline(orc):
    """DF_KINFU_WARPED_INTEGRATE through the frame loop (df_kinfu_*) against the oracle's loop with the same flag, 64^3, 3 frames (two
    warped fusions).  Statistical like tests/test_pipeline_gpu.py: the two solves stop on the reference's PCG tolerance a few per cent
    apart and the field (8 un-normalised translations per voxel) carries that into the fused volume -- and from there into the next
    frame's ICP: by the fourth frame the two pose chains are 5e-3 apart (first GPU run of this test), so the comparison stops at three.
    The bit-for-bit evidence is the stage-level tests above."""
    from dynamicfusion_b200 import kinfu
    from oracle import orc_pipe
    p = kinfu.KinFuParams.default_params_dynamicfusion()
    kinfu.KinFuParams.set_volume(p, 64, 1.0)
    p.max_nodes = 512
    p.cloud_capacity = 400000
    p.flags = kinfu.WARPED_INTEGRATE | kinfu.STAGE_TIMING
    p.fusion_weight_scale = 100.0
    gpu = kinfu.KinFu(p)
    cpu = orc_pipe.KinFu(orc_pipe.params_from(p))
    try:
        for t in range(3):
            depth = synth.umbrella_depth(t)
            assert gpu(depth) == cpu(depth) == (t > 0)
        torch.cuda.synchronize()
        gi, ci = gpu.info(), cpu.info()
        assert gi["nodes"] == ci["nodes"] >= 8 and gi["resets"] == ci["resets"] == 0
        assert gi["n_warped"] > 0 and gi["n_updated"] > 0
        assert gpu.stage_ms()["integrate"] > 0
        assert abs(gi["cloud_points"] - ci["cloud_points"]) <= 0.02 * ci["cloud_points"] + 5, (gi, ci)
        for t in range(3):
            Rg, tg = gpu.getCameraPose(t)
            Rc, tc = cpu.getCameraPose(t)
            assert np.abs(Rg - Rc).max() < 2e-4 and np.abs(tg - tc).max() < 2e-4, t
        vg, vc = gpu.buffer("volume"), cpu.buffer("volume")
        wg, wc = vg >> 16, vc >> 16
        fg = (vg & 0xffff).astype(np.uint16).view(np.float16).astype(np.float32)
        fc = (vc & 0xffff).astype(np.uint16).view(np.float16).astype(np.float32)
        print(f"pipeline (warped integration) after 3 frames: weights differ on {np.mean(wg != wc):.2e}, packed voxels on {np.mean(vg != vc):.2e}")
        assert np.mean(wg != wc) < 2e-2
        same = wg == wc
        assert np.mean(np.abs(fg[same] - fc[same]) > 5e-2) < 2e-2
    finally:
        gpu.close()
        cpu.close()


def test_pipeline_extends_the_field_like_the_oracle_pipeline(orc):
    """DF_KINFU_EXTEND_FIELD through the frame loop against the oracle's loop with the same flag (64^3, 5 frames): the field grows every
    frame; node counts agree within a few nodes (the two clouds differ by a handful of points, see tests/test_pipeline_gpu.py)"""
    from dynamicfusion_b200 import kinfu
    from oracle import orc_pipe
    p = kinfu.KinFuParams.default_params_dynamicfusion()
    kinfu.KinFuParams.set_volume(p, 64, 1.0)
    p.max_nodes = 4096
    p.cloud_capacity = 400000
    p.flags = kinfu.EXTEND_FIELD
    p.extend_radius = 0.05
    gpu = kinfu.KinFu(p)
    cpu = orc_pipe.KinFu(orc_pipe.params_from(p))
    try:
        counts = []
        for t in range(5):
            depth = synth.umbrella_depth(t)
            assert gpu(depth) == cpu(depth) == (t > 0)
            counts.append((gpu.info()["nodes"], cpu.info()["nodes"]))
        print("nodes per frame (gpu, oracle):", counts)
        assert counts[0][0] == counts[0][1] >= 8
        for (g0, c0), (g1, c1) in zip(counts, counts[1:]):
            assert g1 >= g0 and c1 >= c0
        assert counts[-1][0] > counts[0][0] + 20
        for g, c in counts:
            assert abs(g - c) <= max(3, 0.05 * c)
        ng, nc = gpu.buffer("nodes")[: counts[-1][0]], cpu.buffer("nodes")
        M0 = counts[0][0]
        assert np.array_equal(ng[:M0, :3], nc[:M0, :3])
        # appended nodes: identity rotation, weight 3 (their translations have been through the later solves); most of frame 1's
        # additions coincide exactly
        assert np.all(ng[M0:, 3] == 1) and np.all(ng[M0:, 11] == 3) and np.all(ng[M0:, 4:7] == 0)
        # the nodes of the first extension are unsupported by the initial field on both sides (which of the unsupported points were picked
        # depends on every point before them in the cloud, and the two clouds differ by a handful of points: no node-by-node comparison)
        for tab, first in ((ng, counts[1][0]), (nc, counts[1][1])):
            d = np.sqrt(((tab[M0:first, None, :3] - tab[None, :M0, :3]) ** 2).sum(-1)).min(1)
            assert len(d) > 0 and np.all(d > 0.05 * 0.999)
    finally:
        gpu.close()
        cpu.close()
