"""Scenes, image sizes, poses and 6x6 systems for the ICP reference tests (tests/test_icp_float64.py, tests/test_icp_reference_gpu.py).

Image sizes straddle every rule of launch_accumulate (icp.cu): the switch from 256- to 768-thread blocks at 132 x 768 pixels, the block
count below it, ragged rows and partial warps, and HD, where a thread sums 21 pixels.  Scenes: the umbrella and sphere-wall surrogates
(dynamicfusion_b200/synth.py) and four planes whose 6x6 systems reach the solve's branches from image data.  The hook systems feed the
solve tail (df_icp_solve_step) matrices of a chosen spectrum; all their entries are exact float32 values, so the kernel, the reference and
the oracle see the same A.
"""
from __future__ import annotations

import math

import numpy as np

from dynamicfusion_b200 import synth

K = synth.DEFAULT_K
DIST, ANGLE = 0.1, 30 * 0.017453293                      # the frame loop's ICP thresholds (kinfu.cpp)
ITERS = [10, 5, 4]                                        # level 0 (finest) .. 2

# size -> (NT, blocks, k_max) of launch_accumulate
LAUNCH_TABLE = {
    (640, 480): (768, 132, 4),
    (320, 240): (256, 132, 3),
    (160, 120): (256, 75, 1),
    (352, 288): (768, 132, 1),            # exactly 132 x 768 pixels: the first size on 768-thread blocks
    (351, 288): (256, 132, 3),
    (353, 288): (768, 132, 2),
    (203, 151): (256, 120, 1),            # ragged: neither side a multiple of 32
    (7, 5): (256, 1, 1),                  # one block, a partial warp
    (1920, 1080): (768, 132, 21),
}
SIZES = list(LAUNCH_TABLE)


def level_K(K0, level):
    return tuple(k / (1 << level) for k in K0)


# ------------------------------------------------------------------ maps ------------------------------------------------------------------
def maps_points(depth, K0):
    """(vertex, normal) maps of a u16 depth image after the frame loop's bilateral filter (one level)"""
    return pyramid_points(depth, K0, 1)[0]


def maps_depth(depth, K0):
    """(masked depth, normal) of one level: the depth variant's input"""
    return pyramid_depth(depth, K0, 1)[0]


def _depth_levels(depth, levels):
    from oracle import orc
    ds = [orc.bilateral(depth, 7, 4.5, 0.04)]
    for _ in range(levels - 1):
        ds.append(orc.pyr_down(ds[-1], 0.04))
    return ds


def pyramid_points(depth, K0, levels=3):
    """[(vertex, normal)] per level, index 0 finest: bilateral, pyr_down, points_normals (the frame loop's pre-processing)"""
    from oracle import orc
    return [orc.points_normals(level_K(K0, i), d) for i, d in enumerate(_depth_levels(depth, levels))]


def pyramid_depth(depth, K0, levels=3):
    """[(depth, normal)] per level with the depth zeroed where the normal is invalid (computeNormalsAndMaskDepth, kinfu.cpp:241-243)"""
    from oracle import orc
    out = []
    for i, d in enumerate(_depth_levels(depth, levels)):
        n = orc.points_normals(level_K(K0, i), d)[1]
        d = d.copy()
        d[np.isnan(n[..., 0])] = 0
        out.append((d, n))
    return out


# ------------------------------------------------------------------ planes ----------------------------------------------------------------
PLANE_Z0 = 1.0
TILT1 = (0.0, 0.5)                        # Z = z0 + kx X + ky Y: tilted about the image x axis only
TILT2 = (0.3, -0.4)                       # tilted about both axes


def _plane_z(cols, rows, K0, kx, ky, z0):
    fx, fy, cx, cy = K0
    u, v = np.meshgrid(np.arange(cols, dtype=np.float64), np.arange(rows, dtype=np.float64))
    xl, yl = (u - cx) / fx, (v - cy) / fy
    return z0 / (1.0 - kx * xl - ky * yl), xl, yl


def plane_depth(cols, rows, K0, tilt=(0.0, 0.0), z0=PLANE_Z0):
    """u16 millimetre depth of the plane Z = z0 + kx X + ky Y.  (0, 0): fronto-parallel, every normal exactly (0, 0, +-1); (0, ky): the
    depth is constant along image rows, so every normal has an exactly zero x component"""
    z, _, _ = _plane_z(cols, rows, K0, tilt[0], tilt[1], z0)
    return np.clip(np.rint(z * 1000.0), 0, 65535).astype(np.uint16)


def plane_float_maps(cols, rows, K0, tilt=TILT2, z0=PLANE_Z0):
    """the same plane as float vertex and normal maps computed directly (no u16 step, no filtering): the normal is the same float4
    everywhere, so A has rank 3 in exact arithmetic and float rounding leaves its three smallest eigenvalues near zero, of either sign"""
    z, xl, yl = _plane_z(cols, rows, K0, tilt[0], tilt[1], z0)
    v = np.zeros((rows, cols, 4), np.float32)
    v[..., 0], v[..., 1], v[..., 2] = z * xl, z * yl, z
    n = np.array([tilt[0], tilt[1], -1.0]) / math.sqrt(tilt[0] ** 2 + tilt[1] ** 2 + 1.0)
    nm = np.zeros((rows, cols, 4), np.float32)
    nm[..., :3] = n
    return v, nm


# ------------------------------------------------------------------ accumulate cases ------------------------------------------------------
def pose_large():
    """30 degrees about y, 0.3 m sideways and 1 m towards the camera: most points leave the image, part of the cap lands behind the camera
    (s.z <= 0) and projects back into the image, mirrored, onto valid previous points; a few thousand points stay inliers"""
    a = np.deg2rad(30.0)
    R = np.array([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]], np.float32)
    return R, np.array([-0.3, 0.01, -1.0], np.float32)


# pose -> (current frame, T, dist threshold, angle threshold).  The large motion opens both thresholds wide so that what keeps a point
# that lies behind the camera out of the sums is the s.z <= 0 test alone.
POSES = {
    "identity": (0, (np.eye(3, dtype=np.float32), np.zeros(3, np.float32)), DIST, ANGLE),
    "offset": (3, (np.eye(3, dtype=np.float32), np.array([0.002, -0.001, 0.0], np.float32)), DIST, ANGLE),
    "large": (0, pose_large(), 3.0, 80 * 0.017453293),
}


def acc_id(case):
    """the test id of an accumulate case (size, variant, pose)"""
    return f"{case[0][0]}x{case[0][1]}-{case[1]}-{case[2]}"


def accumulate_case(cols, rows, variant, pose):
    """(curr maps, prev maps, K, T, dist2, min_cos): the umbrella at this size; maps are (vertex | depth, normal)"""
    Kl = synth.scaled_K(cols, rows)
    t_curr, T, dist, angle = POSES[pose]
    build = maps_points if variant == "points" else maps_depth
    prev = build(synth.umbrella_depth(0, cols, rows, K=Kl), Kl)
    curr = prev if t_curr == 0 else build(synth.umbrella_depth(t_curr, cols, rows, K=Kl, shape_t=0), Kl)
    return curr, prev, Kl, T, np.float32(dist * dist), np.float32(math.cos(angle))


def oracle_rows(variant, curr, prev, Kl, T, dist2, min_cos):
    from oracle import orc
    fn = orc.icp_rows if variant == "points" else orc.icp_rows_depth
    return fn(curr[0], curr[1], prev[0], prev[1], Kl, T, float(dist2), float(min_cos))


# ------------------------------------------------------------------ estimate scenes -------------------------------------------------------
SCENES = ["umbrella", "sphere-wall", "plane-fronto", "plane-tilt1", "plane-tilt2", "plane-float", "nan-prev"]


def scene_variants(scene):
    return ["points"] if scene == "plane-float" else ["points", "depth"]


def scene_pyramids(scene, variant):
    """(curr pyramid, prev pyramid) at 640 x 480, three levels"""
    pyr = (lambda d: pyramid_points(d, K)) if variant == "points" else (lambda d: pyramid_depth(d, K))
    if scene in ("umbrella", "nan-prev"):
        prev, curr = pyr(synth.umbrella_depth(0)), pyr(synth.umbrella_depth(3, shape_t=0))
        if scene == "nan-prev":                             # no previous surface at the finest level: its first step fails
            v, n = prev[0]
            prev[0] = (np.zeros_like(v) if variant == "depth" else np.full_like(v, np.nan), np.full_like(n, np.nan))
        return curr, prev
    if scene == "sphere-wall":
        return pyr(synth.sphere_wall_depth(seed=1)), pyr(synth.sphere_wall_depth(seed=0))
    if scene == "plane-float":                              # the same frame as source and target
        p = [plane_float_maps(640 >> i, 480 >> i, level_K(K, i)) for i in range(3)]
        return p, p
    tilt = {"plane-fronto": (0.0, 0.0), "plane-tilt1": TILT1, "plane-tilt2": TILT2}[scene]
    return pyr(plane_depth(640, 480, K, tilt, PLANE_Z0 + 0.005)), pyr(plane_depth(640, 480, K, tilt))


def schedule():
    """[(level, iteration within the level)] in execution order: coarse to fine"""
    return [(lvl, i) for lvl in range(len(ITERS) - 1, -1, -1) for i in range(ITERS[lvl])]


def prefix_iters(k):
    """per-level iteration counts (index 0 finest) that run exactly the first k steps of the schedule"""
    it = [0] * len(ITERS)
    for lvl, _ in schedule()[:k]:
        it[lvl] += 1
    return it


# ------------------------------------------------------------------ systems for the solve tail --------------------------------------------
# integer SPD matrices M^T M, M = I + strictly upper integer: det 1, every entry exact, condition numbers by seed (found by search)
SPD_SEEDS = {1e3: (3, 3993), 1e6: (9, 43), 1e8: (9, 3765)}
R_TRUE = np.array([0.01, -0.02, 0.015, 0.003, -0.004, 0.002])


def int_spd(kappa):
    a, seed = SPD_SEEDS[kappa]
    rng = np.random.default_rng(seed)
    M = np.eye(6) + np.triu(rng.integers(-a, a + 1, (6, 6)), 1)
    return M.T @ M


def pack(A, b):
    """the 27 sums of (A, b), float32 values held in float64"""
    A = np.asarray(A, np.float64)
    b = np.asarray(b, np.float64)
    s = np.array([b[i] if j == 6 else A[i, j] for i, j in ((i, j) for i in range(6) for j in range(i, 7))])
    return s.astype(np.float32).astype(np.float64)


def split_table(sums27, nblocks, seed=0):
    """a table of nblocks partial rows whose sum, in any order, is exactly sums27 (float32 values): each entry m 2^e (|m| < 2^24) is split
    into integer multiples of 2^e, so every partial sum is exact in double.  Every row carries a share of the size of the entry itself"""
    rng = np.random.default_rng(seed)
    t = np.zeros((nblocks, 27))
    for s, x in enumerate(np.asarray(sums27, np.float64)):
        if not math.isfinite(x):
            t[:, s] = 0.0
            t[rng.integers(nblocks), s] = x
            continue
        mant, ex = math.frexp(x) if x != 0 else (0.0, 0)
        m, e = int(mant * 2 ** 24), ex - 24
        parts = rng.integers(-(2 ** 22), 2 ** 22, nblocks - 1) if nblocks > 1 else np.zeros(0, np.int64)
        ints = [int(p) for p in parts] + [m - int(sum(int(p) for p in parts))]
        t[:, s] = [math.ldexp(float(i), e) for i in ints]
        assert math.fsum(t[:, s]) == x
    return t


def _hook_systems():
    sc = 64.0                                                   # sums of the size a VGA level gives
    A3 = int_spd(1e3) * sc
    sys_ = {}
    sys_["spd-k1"] = (256.0 * np.eye(6), 256.0 * R_TRUE)
    for kap, name in ((1e3, "spd-k1e3"), (1e6, "spd-k1e6"), (1e8, "spd-k1e8")):
        A = int_spd(kap) * sc
        sys_[name] = (A, A @ R_TRUE)
    Z = A3.copy()
    Z[2, :] = Z[:, 2] = 0.0
    sys_["zero-rowcol"] = (Z, A3 @ R_TRUE)
    for rel, name, r3 in ((1e-14, "tiny-kept", 2.0 ** -7), (1e-16, "tiny-dropped", 2.0 ** 10)):
        T = A3.copy()
        T[3, :] = T[:, 3] = 0.0
        eps = float(np.float32(rel * np.linalg.eigvalsh(T).max()))
        T[3, 3] = eps
        b = T @ R_TRUE
        b[3] = eps * r3                                         # the tiny direction's right-hand side: r_3 = r3 when it is inverted
        sys_[name] = (T, b)
    for side, name in ((1.0, "sI-above"), (-1.0, "sI-below")):  # s^6 = 1e-15 (1 +- 1e-6): on either side of the determinant gate
        s = float(np.float32((1e-15 * (1.0 + side * 1e-6)) ** (1.0 / 6.0)))
        sys_[name] = (s * np.eye(6), s * R_TRUE)
    P = np.eye(6) + np.triu(np.random.default_rng(5).integers(-2, 3, (6, 6)), 1)
    D = np.diag([4.0, 3.0, -2.0, 5.0, 1.0, -6.0]) * sc
    Ind = P.T @ D @ P
    sys_["indefinite"] = (Ind, Ind @ R_TRUE)
    N = A3.copy()
    N[1, 4] = N[4, 1] = np.nan
    sys_["nan-A"] = (N, A3 @ R_TRUE)
    bn = A3 @ R_TRUE
    bn[2] = np.nan
    sys_["nan-b"] = (A3, bn)
    sys_["zeros"] = (np.zeros((6, 6)), np.zeros(6))
    return sys_


HOOK_SYSTEMS = _hook_systems()
# (name, system, table rows): the fixed-order reduction on one row, and on odd and even row counts up to one per SM
HOOK_CASES = [(n, n, 1) for n in HOOK_SYSTEMS] + [(f"spd-k1e3-rows{r}", "spd-k1e3", r) for r in (75, 131, 132)]
BOUNDARY_CASES = {"sI-above", "sI-below"}                  # deliberately 1e-6 from the determinant gate


def hook_T_in():
    from icp_reference import rodrigues
    return rodrigues(np.array([0.1, -0.2, 0.05], np.float32)), np.array([0.3, -0.1, 0.8], np.float32)


def hook_case(name):
    """(sums27, table nblocks x 27, T_in) of one hook case"""
    _, system, rows = next(c for c in HOOK_CASES if c[0] == name)
    sums = pack(*HOOK_SYSTEMS[system])
    return sums, split_table(sums, rows, seed=rows), hook_T_in()
