"""GPU parity: extraction, ICP, k-NN + DQB warp and the data-term solve (through the C ABI) vs the CPU oracle."""
import math

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from dynamicfusion_b200 import host, synth  # noqa: E402

K = synth.DEFAULT_K


def _volume_with_scene(dim, frames=2):
    vol = host.TsdfVolume((dim, dim, dim))
    vol.setTruncDist(0.04); vol.setMaxWeight(64); vol.setSize((1.0, 1.0, 1.0)); vol.setPose(synth.volume_pose(1.0))
    vol.setRaycastStepFactor(0.75); vol.setGradientDeltaFactor(0.5); vol.clear()
    for t in range(frames):
        dists = host.computeDists(host.u16_to_device(synth.umbrella_depth(t, drift=False)), K)
        vol.integrate(dists, host.identity_pose(), K)
    return vol


@pytest.mark.parametrize("dim", [64, 96])
def test_extract_cloud_and_normals(orc, dim):
    vol = _volume_with_scene(dim)
    ref_vol = vol.data_.cpu().numpy().view(np.uint32).copy()
    cap = 400000
    pts, count = vol.fetchCloud(cap)
    n = int(count.item())
    ref = orc.extract_cloud(ref_vol, vol.getDims(), vol.getVoxelSize(), vol.getTruncDist(), vol.getMaxWeight(), vol.getPose(), cap)
    assert n == len(ref) and n > 2000
    got = pts[:n].cpu().numpy()
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), "extraction must match the oracle point for point, in order"
    nrm = vol.fetchNormals(pts, n)
    Rinv = np.linalg.inv(vol.getPose()[0].astype(np.float64)).astype(np.float32)
    ref_n = orc.extract_normals(ref_vol, vol.getDims(), vol.getVoxelSize(), vol.getTruncDist(), vol.getMaxWeight(), ref, vol.getPose(), Rinv, 0.5)
    assert np.array_equal(nrm.cpu().numpy().view(np.uint32), ref_n.view(np.uint32))
    # device-side count path
    nrm2 = vol.fetchNormals(pts, cap, count)[:n]
    assert np.array_equal(nrm2.cpu().numpy().view(np.uint32), ref_n.view(np.uint32))


def test_extract_capacity_clamp_and_empty(orc):
    vol = _volume_with_scene(64)
    pts, count = vol.fetchCloud(1000)
    assert int(count.item()) == 1000
    ref = orc.extract_cloud(vol.data_.cpu().numpy().view(np.uint32).copy(), vol.getDims(), vol.getVoxelSize(), vol.getTruncDist(),
                            vol.getMaxWeight(), vol.getPose(), 1000)
    assert np.array_equal(pts.cpu().numpy().view(np.uint32), ref.view(np.uint32))
    vol.clear()
    pts, count = vol.fetchCloud(1000)
    assert int(count.item()) == 0


def _pyramids(orc, depth):
    d0 = orc.bilateral(depth, 7, 4.5, 0.04)
    ds = [d0]
    for _ in range(2):
        ds.append(orc.pyr_down(ds[-1], 0.04))
    return [orc.points_normals(tuple(k / (1 << i) for k in K), d) for i, d in enumerate(ds)]


def test_icp_accumulate_and_estimate(orc):
    a = _pyramids(orc, synth.umbrella_depth(0))
    b = _pyramids(orc, synth.umbrella_depth(3, shape_t=0))
    icp = host.ProjectiveICP()
    icp.setDistThreshold(0.1); icp.setAngleThreshold(30 * 0.017453293); icp.setIterationsNum([10, 5, 4, 0])
    dev = lambda x: torch.from_numpy(x).cuda()
    T = (np.eye(3, dtype=np.float32), np.array([0.002, -0.001, 0.0], np.float32))
    for lvl in range(3):
        Kl = tuple(k / (1 << lvl) for k in K)
        got = icp.accumulate(dev(b[lvl][0]), dev(b[lvl][1]), dev(a[lvl][0]), dev(a[lvl][1]), Kl, T).cpu().numpy()
        ref, inl = orc.icp_accumulate(b[lvl][0], b[lvl][1], a[lvl][0], a[lvl][1], Kl, T, 0.1 * 0.1, math.cos(30 * 0.017453293))
        assert inl > 1000
        scale = np.abs(ref).max()
        assert np.abs(got - ref).max() <= 1e-5 * scale, (lvl, got - ref)
    ok, (R, t) = icp.estimateTransform(K, [dev(x[0]) for x in b], [dev(x[1]) for x in b], [dev(x[0]) for x in a], [dev(x[1]) for x in a])
    ok_r, (Rr, tr) = orc.icp_estimate([x[0] for x in b], [x[1] for x in b], [x[0] for x in a], [x[1] for x in a], [10, 5, 4], K, 0.1,
                                      np.float32(30 * 0.017453293))
    assert ok and ok_r
    assert np.abs(R - Rr).max() < 1e-5 and np.abs(t - tr).max() < 1e-5
    # run-to-run determinism of the device path
    ok2, (R2, t2) = icp.estimateTransform(K, [dev(x[0]) for x in b], [dev(x[1]) for x in b], [dev(x[0]) for x in a], [dev(x[1]) for x in a])
    assert np.array_equal(R, R2) and np.array_equal(t, t2)


def _depth_pyramids(orc, depth):
    """depth pyramid + normals, depth masked where the normal is invalid (computeNormalsAndMaskDepth, kinfu.cpp:241-243)"""
    d0 = orc.bilateral(depth, 7, 4.5, 0.04)
    ds = [d0]
    for _ in range(2):
        ds.append(orc.pyr_down(ds[-1], 0.04))
    out = []
    for i, d in enumerate(ds):
        n = orc.points_normals(tuple(k / (1 << i) for k in K), d)[1]
        d = d.copy()
        d[np.isnan(n[..., 0])] = 0
        out.append((d, n))
    return out


def test_icp_depth_variant_accumulate_and_estimate(orc):
    """the reference's compile-time USE_DEPTH alternative (proj_icp.cu:47-78, projective_icp.cpp:126-167) vs the oracle, whose
    restatement is pinned bit-exactly to the reference's own USE_DEPTH build (tests/test_oracle_vs_reference_kernels.py)"""
    a = _depth_pyramids(orc, synth.umbrella_depth(0))
    b = _depth_pyramids(orc, synth.umbrella_depth(3, shape_t=0))
    icp = host.ProjectiveICP()
    icp.setDistThreshold(0.1); icp.setAngleThreshold(30 * 0.017453293); icp.setIterationsNum([10, 5, 4, 0])
    dev = lambda x: host.u16_to_device(x) if x.dtype == np.uint16 else torch.from_numpy(x).cuda()
    T = (np.eye(3, dtype=np.float32), np.array([0.002, -0.001, 0.0], np.float32))
    for lvl in range(3):
        Kl = tuple(k / (1 << lvl) for k in K)
        got = icp.accumulateDepth(dev(b[lvl][0]), dev(b[lvl][1]), dev(a[lvl][0]), dev(a[lvl][1]), Kl, T).cpu().numpy()
        ref, inl = orc.icp_accumulate_depth(b[lvl][0], b[lvl][1], a[lvl][0], a[lvl][1], Kl, T, 0.1 * 0.1, math.cos(30 * 0.017453293))
        assert inl > 1000
        scale = np.abs(ref).max()
        assert np.abs(got - ref).max() <= 1e-5 * scale, (lvl, got - ref)
        pts, _ = orc.icp_accumulate(*[orc.points_normals(Kl, x[0])[i] for x, i in ((b[lvl], 0), (b[lvl], 1), (a[lvl], 0), (a[lvl], 1))],
                                    Kl, T, 0.1 * 0.1, math.cos(30 * 0.017453293))
        assert np.abs(pts[26] - ref[26]) > 1e-3 * abs(ref[26])       # not the points variant: the b column differs
    args = ([dev(x[0]) for x in b], [dev(x[1]) for x in b], [dev(x[0]) for x in a], [dev(x[1]) for x in a])
    ok, (R, t) = icp.estimateTransformDepth(K, *args)
    ok_r, (Rr, tr) = orc.icp_estimate_depth([x[0] for x in b], [x[1] for x in b], [x[0] for x in a], [x[1] for x in a], [10, 5, 4], K, 0.1,
                                            np.float32(30 * 0.017453293))
    assert ok and ok_r
    assert np.abs(R - Rr).max() < 1e-5 and np.abs(t - tr).max() < 1e-5
    ok2, (R2, t2) = icp.estimateTransformDepth(K, *args)
    assert np.array_equal(R, R2) and np.array_equal(t, t2)
    blank = [(np.zeros_like(x[0]), x[1]) for x in b]
    ok3, _ = icp.estimateTransformDepth(K, [dev(x[0]) for x in blank], [dev(x[1]) for x in blank], args[2], args[3])
    assert ok3 is False


def test_icp_degenerate_returns_false(orc):
    a = _pyramids(orc, synth.umbrella_depth(0))
    blank = _pyramids(orc, np.zeros((480, 640), np.uint16))
    icp = host.ProjectiveICP()
    dev = lambda x: torch.from_numpy(x).cuda()
    ok, _ = icp.estimateTransform(K, [dev(x[0]) for x in blank], [dev(x[1]) for x in blank], [dev(x[0]) for x in a], [dev(x[1]) for x in a])
    assert ok is False


def _random_nodes(rng, M):
    pts = rng.uniform(-0.3, 0.3, (M, 3)).astype(np.float32)
    nodes = np.zeros((M, 12), np.float32)
    nodes[:, 0:3] = pts
    # random unit rotations + translations, encoded as the reference does (dual = 0.5 * (0,t) * r)
    q = rng.normal(size=(M, 4)).astype(np.float32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    q[:, 0] = np.abs(q[:, 0]) + 1.0                      # keep rotations in one hemisphere (no antipodal cancellation)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    nodes[:, 3:7] = q
    nodes[:, 11] = rng.uniform(0.05, 3.0, M).astype(np.float32)
    return nodes


@pytest.mark.parametrize("M,N", [(8, 100), (300, 5000), (2500, 20000)])
def test_knn_and_warp(orc, M, N):
    import ctypes as C
    rng = np.random.default_rng(M)
    nodes = _random_nodes(rng, M)
    for m in range(M):
        t = rng.normal(scale=0.02, size=3).astype(np.float32)
        orc.load().orc_node_encode_translation(C.c_void_p(nodes[m].ctypes.data), C.c_float(t[0]), C.c_float(t[1]), C.c_float(t[2]))
    if M > 20:
        nodes[10, :3] = nodes[11, :3]                    # duplicate vertex -> distance ties
    pts = rng.uniform(-0.35, 0.35, (N, 4)).astype(np.float32)
    pts[:, 3] = 0
    nrm = rng.normal(size=(N, 4)).astype(np.float32)
    pts[::13, 0] = np.nan
    nrm[::17, 0] = np.nan
    pts[1, :3] = nodes[min(10, M - 1), :3]               # query exactly on a (possibly duplicated) node
    # a third of the queries far outside the node cloud (up to ~1.5 m away, whole warps of them and isolated ones): the grid
    # walk gives up after a few shells and answers them by an exhaustive pass -- same (distance, index) ranking
    far = np.zeros(N, bool); far[N // 2: N // 2 + N // 3] = True; far[5::97] = True
    pts[far, :3] += rng.uniform(0.4, 0.9, (int(far.sum()), 3)).astype(np.float32) * rng.choice([-1.0, 1.0], (int(far.sum()), 3)).astype(np.float32)
    ridx, rd2 = orc.knn8(nodes, pts)
    for use_grid in (False, True):                       # exhaustive shared-memory scan and uniform node grid: identical results
        wf = host.WarpField(use_grid=use_grid)
        wf.setNodes(torch.from_numpy(nodes).cuda())
        idx, d2 = wf.KNN(torch.from_numpy(pts).cuda())
        assert np.array_equal(idx.cpu().numpy(), ridx), f"k-NN indices must be bit-exact (use_grid={use_grid})"
        assert np.array_equal(d2.cpu().numpy().view(np.uint32), rd2.view(np.uint32))
    for flags in (0, 2):
        p_dev, n_dev = torch.from_numpy(pts).cuda(), torch.from_numpy(nrm).cuda()
        kidx, kw = wf.warp(p_dev, n_dev, flags=flags, want_knn=True)
        p_ref, n_ref = pts.copy(), nrm.copy()
        orc.warp(nodes, p_ref, n_ref, flags=flags)
        gp, gn = p_dev.cpu().numpy(), n_dev.cpu().numpy()
        assert np.array_equal(np.isnan(gp), np.isnan(p_ref)) and np.array_equal(np.isnan(gn), np.isnan(n_ref))
        m = ~np.isnan(p_ref[:, 0])
        np.testing.assert_allclose(gp[m], p_ref[m], rtol=1e-4, atol=1e-6)       # north-star tolerance: 1e-4 relative
        mn = ~np.isnan(n_ref[:, 0])
        np.testing.assert_allclose(gn[mn], n_ref[mn], rtol=1e-4, atol=1e-6)
        assert np.mean(gp[m].view(np.uint32) == p_ref[m].view(np.uint32)) > 0.99   # in practice bit-identical (double exp)
    skipped = np.isnan(pts[:, 0]) | np.isnan(nrm[:, 0])
    assert np.array_equal(p_dev.cpu().numpy()[skipped].view(np.uint32), pts[skipped].view(np.uint32)), "skipped points untouched"


@pytest.mark.parametrize("first_nan_normal,N", [(None, 3000), (700, 3000), (0, 3000), (None, 300_000)],
                         ids=["None", "700", "0", "None-300000"])              # 300,000 points: more than 1024 blocks to scan
def test_warp_reference_normal_cursor(orc, first_nan_normal, N):
    """DF_WARP_REF_NORMAL_INDEX: the reference's cursor (warp_field.cpp:182-194) pairs the j-th non-NaN point with normal j and stalls
    for good at the first NaN normal -- with a NaN normal at index 0 (a ray-cast miss at pixel 0) it warps nothing at all"""
    import ctypes as C
    rng = np.random.default_rng(7)
    M = 300
    nodes = _random_nodes(rng, M)
    for m in range(M):
        t = rng.normal(scale=0.02, size=3).astype(np.float32)
        orc.load().orc_node_encode_translation(C.c_void_p(nodes[m].ctypes.data), C.c_float(t[0]), C.c_float(t[1]), C.c_float(t[2]))
    pts = rng.uniform(-0.35, 0.35, (N, 4)).astype(np.float32)
    pts[:, 3] = 0
    nrm = rng.normal(size=(N, 4)).astype(np.float32)
    pts[::7, 0] = np.nan
    pts[100:400, 0] = np.nan                              # whole blocks of invalid points
    if first_nan_normal is not None:
        nrm[first_nan_normal, 0] = np.nan
    wf = host.WarpField()
    wf.setNodes(torch.from_numpy(nodes).cuda())
    p_dev, n_dev = torch.from_numpy(pts).cuda(), torch.from_numpy(nrm).cuda()
    wf.warp(p_dev, n_dev, flags=1)
    p_ref, n_ref = pts.copy(), nrm.copy()
    orc.warp(nodes, p_ref, n_ref, flags=1)
    gp, gn = p_dev.cpu().numpy(), n_dev.cpu().numpy()
    touched_ref = np.any(p_ref.view(np.uint32) != pts.view(np.uint32), axis=1)
    touched_gpu = np.any(gp.view(np.uint32) != pts.view(np.uint32), axis=1)
    assert np.array_equal(touched_ref, touched_gpu)
    valid = int((~np.isnan(pts[:, 0])).sum())
    want = valid if first_nan_normal is None else min(valid, first_nan_normal)
    assert int(touched_ref.sum()) == want
    assert np.array_equal(np.isnan(gp), np.isnan(p_ref)) and np.array_equal(np.isnan(gn), np.isnan(n_ref))
    m = ~np.isnan(p_ref[:, 0])
    np.testing.assert_allclose(gp[m], p_ref[m], rtol=1e-4, atol=1e-6)
    mn = ~np.isnan(n_ref[:, 0])
    np.testing.assert_allclose(gn[mn], n_ref[mn], rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("use_grid,max_nodes,cap", [(True, 4096, 24000), (False, 4096, 24000), (True, 330, 24000), (True, 16384, 330_000)],
                         ids=["True-4096", "False-4096", "True-330", "True-16384-330000"])    # 275,000 points: past the first 1024 blocks
def test_extend_field_matches_oracle(orc, use_grid, max_nodes, cap):
    """df_extend_field (SURVEY 8f(3)): same appended nodes, bit for bit, as the oracle's sequential restatement -- the support test is
    the exact nearest-node distance and the subsampling follows cloud order"""
    rng = np.random.default_rng(11)
    M, P = 300, cap * 5 // 6
    nodes = _random_nodes(rng, M)
    nodes[:, :3] *= 0.5                                    # nodes cover the centre of the cloud only
    cloud = np.zeros((cap, 4), np.float32)
    cloud[:, :3] = rng.uniform(-0.45, 0.45, (cap, 3))
    cloud[::19, 1] = np.nan
    want = orc.extend_field(nodes, cloud[:P], 0.06, 50, max_nodes)
    wf = host.WarpField(use_grid=use_grid)
    wf.setNodes(torch.from_numpy(nodes).cuda())
    count = torch.tensor([P], dtype=torch.int32, device="cuda")
    Mn = wf.extend(torch.from_numpy(cloud).cuda(), 0.06, 50, max_nodes, count)
    got = wf.getNodes().cpu().numpy()
    assert Mn == len(want) == len(got) and (Mn > M + 20 if max_nodes > 1000 else Mn == max_nodes)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    # nothing to add when every point is supported
    assert wf.extend(torch.from_numpy(cloud).cuda(), 10.0, 50, max_nodes + 10, count) == Mn


CUBE = [(1, 1, 1), (1, 1, -1), (1, -1, 1), (1, -1, -1), (-1, 1, 1), (-1, 1, -1), (-1, -1, 1), (-1, -1, -1)]


def _gpu_solve(node_pts, src, dst, nl=300, lin=250, flags=0):
    wf = host.WarpField()
    wf.init(node_pts)
    s = np.zeros((len(src), 4), np.float32); s[:, :3] = src
    d = np.zeros((len(dst), 4), np.float32); d[:, :3] = dst
    # the reference's tests run numIter = 20 outer passes of nonLinearIter = 15 LM steps; every pass re-initialises the
    # trust region (Opt_ProblemInit), which keeps the LM damping away from the rank-deficient systems' null space
    passes = max(1, nl // 15)
    first = None
    for _ in range(passes):
        stats = wf.optimiseWarpData(torch.from_numpy(s).cuda(), torch.from_numpy(d).cuda(), min(nl, 15), lin, flags)
        if first is None:
            first = stats.clone()
    stats[0] = first[0]
    nrm = np.zeros_like(s); nrm[:, 2] = 1
    p_dev, n_dev = torch.from_numpy(s.copy()).cuda(), torch.from_numpy(nrm).cuda()
    wf.warp(p_dev, n_dev)
    return wf, p_dev.cpu().numpy()[:, :3], stats.cpu().numpy()


def test_solve_reference_scenario_single_vertex():
    """reference tests/warp_test.cpp:15-69: 8 cube-corner nodes, one vertex, tolerance 1e-5; closed form 0.05/(8w)"""
    wf, warped, stats = _gpu_solve(CUBE, [(0, 0, 0)], [(0.05, 0.05, 0.05)], nl=15 * 20, lin=250)
    np.testing.assert_allclose(warped, [[0.05, 0.05, 0.05]], atol=1e-5)
    nodes = wf.nodes_.cpu().numpy()
    w = math.exp(-3.0 / 18.0)
    np.testing.assert_allclose(2 * nodes[:, 8:11], np.full((8, 3), 0.05 / (8 * w)), rtol=1e-4)   # identity rotation: t = 2*dual.xyz


@pytest.mark.parametrize("name", ["rigid", "multiple_nodes", "non_rigid"])
def test_solve_reference_scenarios_match_oracle(orc, name):
    from warp_scenarios import SCENARIOS, lsq_reference
    node_pts, src, dst = SCENARIOS[name]
    wf, warped, stats = _gpu_solve(node_pts, src, dst)
    best, _, _ = lsq_reference(node_pts, src, dst)
    np.testing.assert_allclose(warped, best, atol=2e-4)
    nodes_ref = orc.make_nodes(node_pts)
    ostats = orc.solve_data_term(nodes_ref, np.array(src, np.float32), np.array(dst, np.float32), lm_iters=300)
    assert abs(stats[1] - ostats[1]) <= 1e-4 * max(ostats[1], 1e-12) + 1e-10
    assert abs(stats[0] - ostats[0]) <= 1e-9 * ostats[0]
    assert stats[5] == 0


def test_solve_large_matches_matrix_free_oracle(orc):
    from oracle import orc_pipe
    rng = np.random.default_rng(7)
    M, N = 600, 40000
    node_pts = rng.uniform(-0.3, 0.3, (M, 3)).astype(np.float32)
    src = np.zeros((N, 4), np.float32)
    src[:, :3] = rng.uniform(-0.3, 0.3, (N, 3))
    dst = src.copy()
    dst[:, :3] += (0.01 * np.stack([np.sin(5 * src[:, 0]), np.cos(4 * src[:, 1]), src[:, 2]], 1)).astype(np.float32)
    src[::50, 1] = np.nan
    dst[::77, 2] = np.nan
    for flags in (0, 1):
        wf = host.WarpField()
        wf.init(node_pts)
        stats = wf.optimiseWarpData(torch.from_numpy(src).cuda(), torch.from_numpy(dst).cuda(), 5, 100, flags).cpu().numpy()
        nodes_ref = orc.make_nodes(node_pts)
        ostats = orc_pipe.solve_data_term_big(nodes_ref, src, dst, flags=flags, lm_iters=5, lin_iters=100)
        assert stats[3] == ostats[3] and stats[5] == 0
        assert abs(stats[0] - ostats[0]) <= 1e-6 * ostats[0]
        assert abs(stats[1] - ostats[1]) <= 1e-4 * ostats[1]
        got = wf.nodes_.cpu().numpy()
        t_got, t_ref = 2 * got[:, 8:11], orc.node_translations(nodes_ref)[:, 1:]
        assert np.abs(t_got - t_ref).max() <= 1e-3 * np.abs(t_ref).max()


def test_solve_row_overflow_is_loud_and_leaves_the_field_unchanged():
    """ADVICE r1 (solve.cu ROWCAP): a node row that couples to more columns than the kernels store must not be solved truncated.  One
    node at the centre of a sphere of 700 others, 60k vertices at 0.45 R in random directions: every vertex's nearest node is the
    central one, its other seven are the sphere nodes in its direction -- the central node's row couples to (nearly) all 700 columns
    > 512.  Expected: stats[5] raised, 0 LM iterations, the node table bit-identical to its input."""
    rng = np.random.default_rng(11)
    M, N = 701, 60000
    d = rng.normal(size=(M - 1, 3))
    node_pts = np.concatenate([np.zeros((1, 3)), 0.5 * d / np.linalg.norm(d, axis=1, keepdims=True)]).astype(np.float32)
    v = rng.normal(size=(N, 3))
    src = np.zeros((N, 4), np.float32)
    src[:, :3] = 0.45 * 0.5 * v / np.linalg.norm(v, axis=1, keepdims=True)
    dst = src.copy()
    dst[:, 0] += 0.01
    wf = host.WarpField()
    wf.init(node_pts)
    before = wf.nodes_.clone()
    stats = wf.optimiseWarpData(torch.from_numpy(src).cuda(), torch.from_numpy(dst).cuda(), 5, 100, 0).cpu().numpy()
    assert stats[5] == 1 and stats[2] == 0
    assert torch.equal(before, wf.nodes_)


@pytest.mark.parametrize("env", [{"DF_SOLVE_LM_IMPL": "5", "DF_SOLVE_MERGED": "0"}, {"DF_SOLVE_LM_IMPL": "5", "DF_SOLVE_BALANCED": "0"},
                                 {"DF_SOLVE_V6_FORCE_FALLBACK": "1"}, {"DF_SOLVE_LM_IMPL": "1"}, {"DF_SOLVE_LM_CTAS": "8"}])
def test_alternative_icp_and_solve_kernels_in_subprocess(env):
    """The variants that are selected once per process: the v5 cluster LM
    (two exchanges per PCG step) with two reductions per step / fixed lanes per row, v5 as the fallback the default v6 kernel hands a frame
    to when its halo tables do not fit, the one-block LM fallback and the 8-CTA cluster.  Each re-runs this file's ICP / solve parity tests under
    the switch in a fresh interpreter."""
    import os, subprocess, sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_stages_gpu.py", "-q", "-x", "-m", "gpu", "-k",
                        "icp_accumulate_and_estimate or icp_depth or icp_degenerate or solve_reference or solve_large or solve_row_overflow or knn"],
                       cwd=root, env=dict(os.environ, **env), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and "failed" not in r.stdout


def _image_problem(coherent, cols=256, rows=160, M=600, seed=3):
    """an image-shaped solve: canonical vertices on a smooth height field (neighbouring pixels see the same nodes) or scattered at random
    (every tile sees hundreds of nodes: the tile assembly must hand the frame to the per-entry kernels)"""
    rng = np.random.default_rng(seed)
    N = cols * rows
    if coherent:
        u, v = np.meshgrid(np.linspace(-0.3, 0.3, cols), np.linspace(-0.2, 0.2, rows))
        pts = np.stack([u, v, 0.05 * np.sin(6 * u) * np.cos(5 * v)], -1).reshape(N, 3)
        node_pts = pts[rng.choice(N, M, replace=False)].astype(np.float32)
    else:
        pts = rng.uniform(-0.3, 0.3, (N, 3))
        node_pts = rng.uniform(-0.3, 0.3, (M, 3)).astype(np.float32)
    if coherent == "band":                                      # every 8th pixel of 16 image rows lands somewhere else: those tiles see ~140 nodes
        jit = np.zeros(N, bool)                                 # (more than a record holds -> redone as pixel-row records), their strips ~25
        jit[80 * cols:96 * cols:8] = True
        pts[jit] += rng.uniform(-0.15, 0.15, (int(jit.sum()), 3))
    src = np.zeros((N, 4), np.float32)
    src[:, :3] = pts
    dst = src.copy()
    dst[:, :3] += (0.01 * np.stack([np.sin(5 * src[:, 0]), np.cos(4 * src[:, 1]), src[:, 2]], 1)).astype(np.float32)
    src[7::50, 1] = np.nan                                      # (vertex 0 stays valid: the graph quirk hangs its extra edges on it)
    dst[11::77, 2] = np.nan
    src[40 * cols:48 * cols, 0] = np.nan                        # a band of empty tiles
    return node_pts, src, dst, cols


@pytest.mark.parametrize("coherent", [True, False, "band"])
def test_solve_tile_assembly_matches_per_entry_path_and_oracle(orc, coherent):
    """DF_SOLVE_IMAGE_COLS: the normal matrix assembled from 16 x 8-pixel tile records (round 2) against the per-entry kernels (same
    solve from a flat vertex list) and against the matrix-free oracle.  stats[7]'s fraction tells which path built the matrix."""
    from oracle import orc_pipe
    node_pts, src, dst, cols = _image_problem(coherent)
    out = {}
    for name, flags in (("flat", 0), ("tiles", cols << 8), ("tiles_quirk", (cols << 8) | 1), ("flat_quirk", 1)):
        wf = host.WarpField()
        wf.init(node_pts)
        stats = wf.optimiseWarpData(torch.from_numpy(src).cuda(), torch.from_numpy(dst).cuda(), 5, 100, flags).cpu().numpy()
        out[name] = (stats, wf.nodes_.cpu().numpy())
        assert stats[5] == 0
        used_tiles = abs(stats[7]) % 1 == 0.5
        assert used_tiles == (bool(coherent) and name.startswith("tiles")), (name, stats)
    for a, b in (("flat", "tiles"), ("flat_quirk", "tiles_quirk")):
        sa, na = out[a]; sb, nb = out[b]
        assert sa[3] == sb[3] and sa[2] == sb[2]
        assert abs(sa[0] - sb[0]) <= 1e-12 * abs(sa[0]) and abs(sa[1] - sb[1]) <= 1e-9 * abs(sa[1])
        assert sa[6] >= sb[6]                                      # the tile path drops exact-zero products, nothing else
        t_a, t_b = 2 * na[:, 8:11], 2 * nb[:, 8:11]
        assert np.abs(t_a - t_b).max() <= 1e-4 * np.abs(t_a).max()
    nodes_ref = orc.make_nodes(node_pts)
    ostats = orc_pipe.solve_data_term_big(nodes_ref, src, dst, flags=0, lm_iters=5, lin_iters=100)
    stats, got = out["tiles"]
    assert stats[3] == ostats[3]
    assert abs(stats[0] - ostats[0]) <= 1e-6 * ostats[0] and abs(stats[1] - ostats[1]) <= 1e-4 * ostats[1]
    t_got, t_ref = 2 * got[:, 8:11], orc.node_translations(nodes_ref)[:, 1:]
    assert np.abs(t_got - t_ref).max() <= 1e-3 * np.abs(t_ref).max()


@pytest.mark.parametrize("cols,rows", [(256, 160), (200, 100)])
def test_knn_on_image_shaped_queries(orc, cols, rows):
    """The 8-NN grid walk (knn8_grid) on queries that are neighbours in the image, which the random point sets of test_knn_and_warp never
    produce, against the oracle's exhaustive search: indices and squared distances bit for bit, through df_knn8 (32 consecutive queries per
    warp) and through df_warp's neighbour output with the 8 x 4 patch mapping of DF_WARP_IMAGE_COLS (256 x 160; 200 x 100 does not qualify
    and keeps the linear map).  Includes duplicated nodes (ties at every rank), NaN pixels, a depth edge (a warp whose queries straddle two
    surfaces) and a far region 0.6 m off the node cloud."""
    rng = np.random.default_rng(cols)
    N = cols * rows
    u, v = np.meshgrid(np.linspace(-0.3, 0.3, cols), np.linspace(-0.2, 0.2, rows))
    z = 0.05 * np.sin(6 * u) * np.cos(5 * v)
    z[:, cols // 2:] += 0.08                                      # a depth edge down the middle of the image
    pts3 = np.stack([u, v, z], -1).reshape(N, 3).astype(np.float32)
    M = 700
    nodes = _random_nodes(rng, M)
    nodes[:, :3] = pts3[rng.choice(N, M, replace=False)]
    nodes[40:48, :3] = nodes[39, :3]                              # nine coincident nodes: ties decide a whole neighbour set
    pts = np.zeros((N, 4), np.float32)
    pts[:, :3] = pts3
    pts[3::29, 0] = np.nan
    far = np.zeros((rows, cols), bool); far[: rows // 8] = True   # the top rows look at a region 0.6 m off the node cloud
    pts[far.reshape(-1), 2] += 0.6
    nrm = np.zeros((N, 4), np.float32); nrm[:, 2] = 1
    ridx, rd2 = orc.knn8(nodes, pts)
    wf = host.WarpField(use_grid=True)
    wf.setNodes(torch.from_numpy(nodes).cuda())
    idx, d2 = wf.KNN(torch.from_numpy(pts).cuda())
    assert np.array_equal(idx.cpu().numpy(), ridx)
    assert np.array_equal(d2.cpu().numpy().view(np.uint32), rd2.view(np.uint32))
    p_dev, n_dev = torch.from_numpy(pts).cuda(), torch.from_numpy(nrm).cuda()
    kidx, kw = wf.warp(p_dev, n_dev, flags=cols << 8, want_knn=True)
    valid = ~np.isnan(pts[:, 0])
    assert np.array_equal(kidx.cpu().numpy()[valid], ridx[valid])
    p_ref, n_ref = pts.copy(), nrm.copy()
    orc.warp(nodes, p_ref, n_ref)
    np.testing.assert_allclose(p_dev.cpu().numpy()[valid], p_ref[valid], rtol=1e-4, atol=1e-6)
