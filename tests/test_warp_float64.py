"""The float64 reference of the warp side (warp_reference.py) against the C oracle, on the CPU: the oracle's k-NN sets must be admissible, its
warped points and normals and its warped-fusion volumes must lie within every bar with few enough ambiguous queries and voxels that the
bars cannot pass by accident, and references perturbed the way a kernel could get the operation wrong (a half-voxel offset, the weight's
exponent without its 1/2, a translation taken without the conjugate rotation, warp_to_live applied before the blend, 7 neighbours, two voxel
sizes swapped, the weight as a mean over the valid neighbours) must land far outside them.  The search-path restatement is checked on the
fusion cases' node layouts."""
import functools

import numpy as np
import pytest

import warp_cases as wc
import warp_reference as wr

pytestmark = pytest.mark.usefixtures("orc")

AMB_MAX = 1e-3
W2L = wc.f32(wc.W2L)


@pytest.mark.parametrize("M", [5, 8, 300, 2500])
def test_oracle_knn_sets_are_admissible(orc, M):
    rng = np.random.default_rng(M)
    nodes = wc.random_nodes(orc, M, M)
    q = wc.queries(rng, 4000)
    idx, d2 = orc.knn8(nodes, q)
    ref = wr.knn64(nodes, wr.f64(q)[:, :3])
    assert np.all(wr.knn_admissible(ref, idx))
    ok = idx >= 0
    V = wr.f64(nodes)[:, :3]
    exact = ((wr.f64(q)[:, None, :3] - V[np.where(ok, idx, 0)]) ** 2).sum(-1)
    assert np.all(np.abs(d2[ok] - exact[ok]) <= wr.KNN_MARGIN * wr.U * exact[ok])
    amb = 1 - ref["forced"].mean()
    print(f"\nknn M={M}: ambiguous queries {amb:.2e}")
    assert amb < AMB_MAX


def test_lattice_ties_are_exact(orc):
    """nodes and queries on a lattice of 2^-6 m: every distance is exact in float32, ties are exact on both sides and the oracle's set is
    the float64 (distance, index) order itself"""
    c = wc.case("lattice")
    nodes = wc.case_nodes(orc, c)
    lin = np.random.default_rng(1).integers(0, 64 ** 3, 5000)
    _, xc, delta, ex = wr.voxel_positions(c["dims"], c["vs"], c["pose_v"], lin)
    assert ex.all() and np.all(delta == 0)
    idx, _ = orc.knn8(nodes, xc.astype(np.float32))
    ref = wr.knn64(nodes, xc, delta, ex)
    assert ref["forced"].all() and np.array_equal(idx, ref["idx"])
    ties = (np.diff(ref["cand_d2"][:, :9], axis=1) == 0).any(1).mean()
    print(f"\nlattice: queries with exact distance ties among their 9 nearest {ties:.2f}")
    assert ties > 0.2


def _warp_oracle(orc, nodes, pts, nrm, w2l, flags):
    p, n = pts.copy(), nrm.copy()
    orc.warp(nodes, p, n, w2l, flags)
    return p, n


@pytest.mark.parametrize("kind", ["trans", "rot3", "rotbig"])
@pytest.mark.parametrize("rotate_only", [False, True])
def test_oracle_warp_lies_within_the_bars(orc, kind, rotate_only):
    rng = np.random.default_rng(7)
    nodes = wc.random_nodes(orc, 400, 4, rotations=False)
    if kind != "trans":
        for i in range(len(nodes)):
            rot = wc.random_rotations(rng, 1)[0] if kind == "rotbig" else wc._quat_axis_angle(rng.normal(size=3), rng.uniform(-3, 3))
            t = rng.normal(scale=0.02, size=3).astype(np.float32)
            wc._encode(orc, nodes, i, t, rot)
    pts = wc.queries(rng, 3000)
    nrm = rng.normal(size=(3000, 4)).astype(np.float32)
    nrm[:, :3] /= np.linalg.norm(nrm[:, :3], axis=1, keepdims=True)
    p, n = _warp_oracle(orc, nodes, pts, nrm, W2L, 2 if rotate_only else 0)
    ref = wr.warp64(nodes, pts, nrm, W2L, rotate_only)
    bad, rp, rn, nchk = wr.warp_check(p, n, ref)
    amb = ref[4].mean()
    print(f"\nwarp {kind} rotate_only={rotate_only}: worst point {rp:.3g} normal {rn:.3g} bars, ambiguous {amb:.2e}")
    assert bad == 0 and nchk > 0.99 * len(pts) and amb < AMB_MAX
    assert rp > 1e-3


# ------------------------------------------------------------------ warped fusion --------------------------------------------------------------
# reduced sizes: every case's field, frame, K, pose and weights on the small volumes
SMALL = ["ragged-weights-tiny", "deep-m5", "lattice", "rotated-w2l", "ragged-rotbig", "ragged-grid"]


def small_case(cid):
    """the case on the 40 x 28 x 36 volume when its own is large; its field, frame, K, pose and weights unchanged"""
    c = wc.case(cid)
    if c["vol"] in ("deep", "aniso", "bench"):
        c.update(vol="ragged", dims=wc.VOLUMES["ragged"][0], vs=wc.voxel_size("ragged"), trunc=wc.trunc_dist("ragged"),
                 pose_v=wc.f32(wc.volume_pose("ragged", c["pose"])))
    return c


def _oracle_passes(orc, c, nodes, passes=None):
    """the oracle's volume after each pass: [(prev, after, depth, world2cam, n)]"""
    vol = np.zeros(int(np.prod(c["dims"])), np.uint32)
    out = []
    for p in range(passes or c["passes"]):
        depth = wc.case_depth(c, p)
        w2c = wc.case_world2cam(c, p)
        prev = vol.copy()
        n = orc.integrate_warped(vol, c["dims"], c["vs"], c["trunc"], c["maxw"], depth, c["pose_v"], w2c, c["K"], nodes, c["ws"])
        out.append((prev, vol.copy(), depth, w2c, n))
    return out


def _check_passes(c, nodes, passes, perturb=None):
    warped = wr.warp_voxels(nodes, c["dims"], c["vs"], c["pose_v"], perturb=perturb)
    res = []
    for prev, vol, depth, w2c, n in passes:
        ref = wr.integrate_warped64(prev, warped, depth, c["K"], w2c, c["trunc"], c["maxw"], c["ws"])
        res.append(wr.integrate_warped_check(prev, vol, ref) + (n,))
    return res, warped


@pytest.mark.parametrize("cid", SMALL)
def test_oracle_integrate_warped_lies_within_the_bars(orc, cid):
    c = small_case(cid)
    nodes = wc.case_nodes(orc, c)
    passes = _oracle_passes(orc, c, nodes)
    res, warped = _check_passes(c, nodes, passes)
    nvox = int(np.prod(c["dims"]))
    for bad, ratio, nupd, namb, n in res:
        print(f"\n{cid}: {bad} outside, worst {ratio:.3g} bars, {nupd} updated + {namb} ambiguous, oracle wrote {n}")
        assert bad == 0
        assert nupd <= n <= nupd + namb
        assert namb / nvox < AMB_MAX * 5
    assert sum(r[2] for r in res) > 500
    if c["maxw"] == 8 and c["ws"] >= 400:                       # both weight clamps reached
        W = passes[-1][1] >> 16
        assert (W == 8).sum() > 100


# which check each perturbation is measured on: the warped-fusion volume of a small case, or df_warp's points and normals under rotated nodes
PERTURBATIONS = {"half_voxel": "integrate", "swap_vsy_vsz": "integrate", "exp_no_half": "both", "k7": "both", "no_conj": "warp",
                 "w2l_first": "warp"}


@functools.lru_cache(maxsize=None)
def _one_pass(cid):
    c = small_case(cid)
    nodes = wc.case_nodes(_orc(), c)
    return c, nodes, _oracle_passes(_orc(), c, nodes, passes=1)


def _orc():
    import oracle.orc as orc
    return orc


@pytest.mark.parametrize("how", list(PERTURBATIONS))
def test_perturbed_references_land_far_outside_the_bars(orc, how, capsys):
    worst = 0.0
    if PERTURBATIONS[how] in ("integrate", "both"):
        c, nodes, passes = _one_pass("ragged-weights-tiny")            # vsx, vsy and vsz all differ
        (bad, ratio, nupd, namb, n), = _check_passes(c, nodes, passes, perturb=how)[0]
        worst = max(worst, ratio)
    if PERTURBATIONS[how] in ("warp", "both"):
        rng = np.random.default_rng(3)
        nodes = wc.random_nodes(orc, 300, 9)
        pts = wc.queries(rng, 2000)
        nrm = rng.normal(size=(2000, 4)).astype(np.float32)
        p, n = _warp_oracle(orc, nodes, pts, nrm, W2L, 0)
        _, rp, rn, _ = wr.warp_check(p, n, wr.warp64(nodes, pts, nrm, W2L, perturb=how))
        worst = max(worst, rp, rn)
    with capsys.disabled():
        print(f"\n{how}: worst {worst:.3g} bars")
    assert worst >= 100


def test_mean_weight_fails_the_exact_weight_check(orc):
    """with M = 5 the weight is sum / 8 over the five nodes, not their mean: the mean's weights are not the oracle's"""
    c, nodes, passes = _one_pass("deep-m5")
    (bad, _, nupd, _, _), = _check_passes(c, nodes, passes)[0]
    assert bad == 0
    (bad, _, nupd, _, _), = _check_passes(c, nodes, passes, perturb="mean_weight")[0]
    print(f"\nmean weight: {bad} of {nupd} voxels outside")
    assert bad > 0.1 * nupd


def test_search_path_restatement():
    """the fusion cases' node layouts take the search path each is built for, by a wide margin"""
    import oracle.orc as orc
    for cid in ("deep-cluster", "coarse-spread", "ragged-grid", "deep-m5", "deep-trans"):
        c = wc.case(cid)
        nodes = wc.case_nodes(orc, c)
        sp = wr.search_path(nodes, c["dims"], c["vs"], c["pose_v"])
        print(f"\n{cid}: list {sp['list']:.2f} tree {sp['tree']:.2f} grid {sp['grid']:.2f}; block lists "
              f"{min(sp['block_n'], default=0)}..{max(sp['block_n'], default=0)}, run lists {min(sp['run_n'], default=0)}..{max(sp['run_n'], default=0)}")
        assert wr.path_of(sp) == c["path"], (cid, wr.path_of(sp))


@pytest.mark.parametrize("cid", list(wc.CASES))
def test_straddling_runs_only_where_built(cid):
    """the visibility cull's camera-plane exit decides for visible voxels in the cases built for it, with a margin of 16 pixels and 0.1 mm"""
    c = wc.case(cid)
    runs = wr.straddle_runs(c["dims"], c["vs"], wc.case_vol2cam(c, 0), c["K"], c["cols"], c["rows"])
    print(f"\n{cid}: straddling runs with voxels in view {runs}")
    assert bool(runs) == (cid in wc.STRADDLE)
    if runs:
        assert sum(n for _, n in runs) >= 8
