"""Shapes of the warp side's float64 tests (k-NN, the DQB warp, per-voxel warped fusion) and the helpers the warped-fusion GPU tests share:
non-cubic volumes with a partial last z-chunk, strongly anisotropic voxels and a rotated volume pose; ragged and pitched frames; intrinsics
with fx != fy and an off-centre principal point; the camera in front of, tilted against and inside the volume; fields with no, small and
large node rotations, node weights on both sides of node_weighting's polynomial range, duplicated vertices, nodes on the voxel lattice, every
node-count regime of the fusion kernel's search (no lists below 8 nodes, no BVH above 8192) and node layouts that overflow its run and block
candidate lists.  CPU only (numpy, synth and the oracle's node encoders)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from dynamicfusion_b200 import synth

K = synth.DEFAULT_K
DEFAULT_K = tuple(float(k) for k in synth.DEFAULT_K)
K2 = (585.0, 548.5, 331.75, 226.25)              # fx != fy, principal point off the image centre
TRUNC, MAXW = 0.04, 64
PITCH_PAD = [0, 2, 512]                           # bytes added to each row of the depth image
FUS_LIST_CAP, FUS_BLOCK_CAP, BVH_MAX_M = 768, 2048, 8192      # csrc/fusion.cu, csrc/warp_common.cuh (NODEGRID_ORDER_MAX_M)


# ------------------------------------------------------------------ helpers shared with test_fusion_gpu.py / test_warped_color_gpu.py ----------
def _volume(dim, size):
    """a tracked dim^3 host.TsdfVolume of edge `size` at synth.volume_pose, truncation TRUNC, maximum weight MAXW"""
    from dynamicfusion_b200 import host
    vol = host.TsdfVolume((dim, dim, dim), track_activity=True)
    vol.setTruncDist(TRUNC)
    vol.setMaxWeight(MAXW)
    vol.setSize((size, size, size))
    vol.setPose(synth.volume_pose(size))
    vol.clear()
    return vol


def _surface_nodes(orc, M, seed, t_scale=0.0, rotate=False, weight=3.0):
    """nodes scattered on the sphere-and-wall scene, with random translations (and optionally rotations) encoded as the reference's
    DualQuaternion(translation, rotation) does"""
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(M, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    v = (np.array([0.0, 0.0, 1.0]) + 0.25 * d).astype(np.float32)
    v[::3, 2] = 1.38                                         # a third of them on the wall
    v[::3, :2] = rng.uniform(-0.45, 0.45, size=(len(v[::3]), 2))
    nodes = orc.make_nodes(v, weight)
    lib = orc.load()
    for i in range(M):
        if rotate:
            ang = rng.uniform(-0.05, 0.05, 3).astype(np.float32)
            t = (rng.uniform(-1, 1, 3) * t_scale).astype(np.float32)
            rot = np.zeros(4, np.float32)
            dual = np.zeros(4, np.float32)
            lib.orc_dq_from_euler(C.c_float(float(t[0])), C.c_float(float(t[1])), C.c_float(float(t[2])), C.c_float(float(ang[0])),
                                  C.c_float(float(ang[1])), C.c_float(float(ang[2])), C.c_void_p(rot.ctypes.data), C.c_void_p(dual.ctypes.data))
            nodes[i, 3:7] = rot
            nodes[i, 7:11] = dual
        elif t_scale > 0:
            t = (rng.uniform(-1, 1, 3) * t_scale).astype(np.float32)
            lib.orc_node_encode_translation(C.c_void_p(nodes[i].ctypes.data), C.c_float(float(t[0])), C.c_float(float(t[1])), C.c_float(float(t[2])))
    return nodes


def _tilted_pose():
    a, b = np.deg2rad(5.0), np.deg2rad(-3.0)
    Rx = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
    Ry = np.array([[np.cos(b), 0, np.sin(b)], [0, 1, 0], [-np.sin(b), 0, np.cos(b)]])
    return (Rx @ Ry).astype(np.float32), np.array([0.02, -0.015, 0.03], np.float32)


# ------------------------------------------------------------------ poses ---------------------------------------------------------------------
def _rot(ax, deg):
    a = np.deg2rad(deg)
    c, s = np.cos(a), np.sin(a)
    if ax == "x":
        return np.array([[1, 0, 0], [0, c, -s], [0, s, c]])
    if ax == "y":
        return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])


def f32(A):
    return np.ascontiguousarray(A[0], np.float32), np.ascontiguousarray(A[1], np.float32)


def _mul(A, B):
    return A[0] @ B[0], A[0] @ B[1] + A[1]


def _inv(A):
    Ri = A[0].T
    return Ri, -Ri @ A[1]


# name: (dims, size in metres, volume rotation); the comment says what the shape exercises
VOLUMES = {
    "deep": ((100, 72, 136), (0.8, 0.576, 1.088), None),          # Dz >= 64: z-chunk 32, last chunk 8; 8 mm voxels
    "aniso": ((96, 64, 72), (0.576, 0.576, 1.008), None),         # voxels of (6, 9, 14) mm; last z-chunk 8
    "rotated": ((64, 64, 64), (0.64, 0.64, 0.64), (10.0, 5.0)),   # volume pose rotated 10 degrees about y and 5 about x
    "aniso60": ((96, 64, 72), (0.576, 0.576, 1.008), (60.0, 0.0)),   # (6, 9, 14) mm voxels at 60 degrees about y: run boxes long and thin
                                                                    # across the view; inside, one straddles the camera plane (STRADDLE)
    "ragged": ((40, 28, 36), (1.0, 1.0, 1.0), None),              # dims no multiple of the 32 x 8 block footprint, one z-chunk
    "lattice": ((64, 64, 64), (1.0, 1.0, 1.0), None),             # voxel size 2^-6 m at synth.volume_pose: positions and distances exact
    "coarse": ((48, 24, 48), (1.92, 0.96, 1.92), None),           # 4 cm voxels: a block's region holds metres of the field
    "bench": ((256, 256, 256), (1.0, 1.0, 1.0), None),            # the bench's volume
}


def voxel_size(name):
    dims, size, _ = VOLUMES[name]
    return (np.asarray(size, np.float32) / np.asarray(dims, np.float32)).astype(np.float32)


def trunc_dist(name):
    """TsdfVolume::setTruncDist's rule: at least 2.1 voxels of the largest voxel size"""
    return float(max(np.float32(TRUNC), np.float32(2.1) * voxel_size(name).max()))


def volume_pose(name, pose_kind):
    """volume-to-world: the volume about the optical axis with its near face 0.5 m in front of the camera, or ('inside') the camera plane
    cutting it at 30 % of its depth.  Offsets of a millimetre or two keep voxel centres off the planes x = 0 and y = 0.  The lattice volume
    keeps synth.volume_pose, whose translation is a multiple of its voxel size."""
    dims, size, rot = VOLUMES[name]
    if name == "lattice":
        R, t = synth.volume_pose(size[0])
        return np.asarray(R, np.float64), np.asarray(t, np.float64)
    z0 = -0.3 * size[2] if pose_kind == "inside" else 0.5
    t = np.array([-size[0] / 2 + 0.00137, -size[1] / 2 - 0.00091, z0 + 0.00213])
    if rot is None:
        return np.eye(3), t
    R = _rot("y", rot[0]) @ _rot("x", rot[1])
    centre = t + 0.5 * np.asarray(size)
    return R, centre - R @ (0.5 * np.asarray(size)) + np.asarray(STRADDLE_SHIFT.get((name, pose_kind), (0.0, 0.0, 0.0)))


# The visibility cull of csrc/fusion.cu projects a run box's eight corners, and it must not reason projectively about a box that straddles
# the camera plane: behind the camera the projection flips sign, so all eight corners can fall on one side of the image while voxels of the
# box in front of the camera project into it.  For an axis-aligned box that cannot happen; for a long, thin box at an angle to the view it
# can.  This shift of the 60-degree volume puts one run of 8 x 4 x 8 voxels around the camera in exactly that configuration, with voxels in
# front of it that the frame updates (warp_reference.straddle_runs finds them): only the cull's camera-plane exit keeps them.
STRADDLE_SHIFT = {("aniso60", "inside"): (0.0188, 0.0212, 0.0058)}
STRADDLE = {"aniso60-inside"}                     # cases whose updated voxels include some that only the camera-plane exit keeps


def camera_pose(pose_kind):
    """camera-to-world of the first pass"""
    if pose_kind in ("front", "inside"):
        return np.eye(3), np.zeros(3)
    assert pose_kind == "tilted"
    return _rot("x", 5.0) @ _rot("y", -3.0), np.array([0.02, -0.015, 0.03])


def pass_pose(pose_kind, p):
    """camera-to-world of pass p: the case's pose, then small moves (the running average sees different samples)"""
    moves = [(np.eye(3), np.zeros(3)), (np.eye(3), np.array([0.003, 0.0, 0.002])), (_rot("y", 0.4), np.array([-0.003, 0.002, 0.0]))]
    return _mul(camera_pose(pose_kind), moves[p])


W2L = (_rot("z", 2.0) @ _rot("x", -1.5), np.array([0.004, -0.003, 0.006]))       # a non-identity warp_to_live


def world2cam(pose_kind, p, w2l=False):
    """inv(camera pose) . warp_to_live, as host.TsdfVolume.integrate_warped composes it"""
    A = _inv(pass_pose(pose_kind, p))
    return f32(_mul(A, W2L) if w2l else A)


def scene(name, pose_kind):
    """(sphere centre, radius, wall z) of the depth scene: a sphere in front of a wall inside the volume's depth range"""
    dims, size, _ = VOLUMES[name]
    if name == "aniso60":
        return np.array([0.02, -0.01, 0.3]), 0.1, 0.6
    lo = max(volume_pose(name, pose_kind)[1][2], 0.08) if VOLUMES[name][2] is None else 0.55
    hi = volume_pose(name, "front" if pose_kind != "inside" else "inside")[1][2] + size[2] - (0.05 if VOLUMES[name][2] else 0.0)
    r = 0.3 * min(size[0], size[1], hi - lo)
    return np.array([0.02, -0.01, lo + 0.45 * (hi - lo)]), r, lo + 0.93 * (hi - lo)     # the wall inside the last z-chunk


def scene_depth(name, pose_kind, cols, rows, K, p):
    c, r, wall = scene(name, pose_kind)
    return synth.sphere_wall_depth(cols=cols, rows=rows, K=K, seed=1000 * p + cols, radius=r, centre=tuple(c), wall_z=wall)


def frame_K(kind, cols, rows):
    """K scaled from 640 x 480 to the frame"""
    K0 = DEFAULT_K if kind == "default" else K2
    return (K0[0] * cols / 640.0, K0[1] * rows / 480.0, K0[2] * cols / 640.0, K0[3] * rows / 480.0)


# ------------------------------------------------------------------ fields --------------------------------------------------------------------
def _encode(orc, nodes, i, t, rot=None):
    """node i: translation t (and rotation quaternion rot), encoded as the reference's DualQuaternion(translation, rotation) does"""
    lib = orc.load()
    if rot is not None:
        nodes[i, 3:7] = rot
    lib.orc_node_encode_translation(C.c_void_p(nodes[i].ctypes.data), C.c_float(float(t[0])), C.c_float(float(t[1])), C.c_float(float(t[2])))


def _on_scene(rng, M, name, pose_kind):
    """M points on the case's sphere (two thirds) and wall (one third), in world coordinates"""
    c, r, wall = scene(name, pose_kind)
    d = rng.normal(size=(M, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    v = c + r * d
    size = VOLUMES[name][1]
    v[::3, 2] = wall
    v[::3, :2] = rng.uniform(-0.45, 0.45, size=(len(v[::3]), 2)) * np.asarray(size[:2])
    return v.astype(np.float32)


def _quat_axis_angle(axis, deg):
    a = np.deg2rad(deg) / 2
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    return np.concatenate([[np.cos(a)], np.sin(a) * axis]).astype(np.float32)


def random_rotations(rng, M):
    """large random rotations in one hemisphere (no antipodal cancellation in the blend), as the stage tests make them"""
    q = rng.normal(size=(M, 4)).astype(np.float32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    q[:, 0] = np.abs(q[:, 0]) + 1.0
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    return q.astype(np.float32)


def random_nodes(orc, M, seed, rotations=True):
    """M nodes in a 0.6 m cube: large rotations in one hemisphere (unless rotations is False), translations of 2 cm, node weights from 0.05
    to 3 and, from 21 nodes on, one duplicated vertex"""
    rng = np.random.default_rng(seed)
    nodes = orc.make_nodes(rng.uniform(-0.3, 0.3, (M, 3)).astype(np.float32), 3.0)
    if rotations:
        nodes[:, 3:7] = random_rotations(rng, M)
    nodes[:, 11] = rng.uniform(0.05, 3.0, M).astype(np.float32)
    for m in range(M):
        _encode(orc, nodes, m, rng.normal(scale=0.02, size=3).astype(np.float32))
    if M > 20:
        nodes[10, :3] = nodes[11, :3]
    return nodes


def queries(rng, N):
    """N query points [N, 4] in and around random_nodes' cube, a twentieth of them far outside it (the grid walk's BVH fallback)"""
    q = np.zeros((N, 4), np.float32)
    q[:, :3] = rng.uniform(-0.35, 0.35, (N, 3))
    q[:N // 20, :3] *= 8.0
    return q


def field(orc, kind, M, name, pose_kind, seed):
    """the node table [M, 12] of a field kind on the case's scene:
      identity   no motion;
      trans      translations of +-2 mm, three rim nodes moving by decimetres (the global displacement bound culls nothing);
      rot3       rotations of up to 3 degrees about random axes and translations of +-2 mm;
      rotbig     large random rotations in one hemisphere and translations of +-5 mm;
      weights    translations of +-2 mm, node weights from 0.05 to 3 (both exp paths of node_weighting) and duplicated vertices;
      lattice    nodes on voxel centres of the lattice volume (exact float64 ties between equidistant nodes), translations of +-2 mm;
      cluster    every node within 1.5 cm of the sphere's front point (every run's candidate list overflows, the block list fits);
      spread     nodes filling the coarse volume (its block lists overflow)"""
    rng = np.random.default_rng(seed)
    if kind == "lattice":
        dims = np.asarray(VOLUMES[name][0])
        R, t = volume_pose(name, pose_kind)
        vs = voxel_size(name).astype(np.float64)
        g = rng.integers(4, dims - 4, size=(M, 3))
        v = (R @ (g * vs).T).T + t
    elif kind == "cluster":
        c, r, _ = scene(name, pose_kind)
        v = c - np.array([0.0, 0.0, r]) + rng.uniform(-0.015, 0.015, size=(M, 3))
    elif kind == "spread":
        R, t = volume_pose(name, pose_kind)
        size = np.asarray(VOLUMES[name][1])
        v = (R @ (rng.uniform(0.05, 0.95, size=(M, 3)) * size).T).T + t
    else:
        v = _on_scene(rng, M, name, pose_kind)
    nodes = orc.make_nodes(np.asarray(v, np.float32), 3.0)
    if kind == "weights":
        nodes[:, 11] = rng.uniform(0.05, 3.0, M).astype(np.float32)
        nodes[1::7, :3] = nodes[0::7, :3][: len(nodes[1::7])]            # duplicated vertices: distance ties between distinct nodes
    if kind == "identity":
        return nodes
    for i in range(M):
        rot = None
        if kind == "rot3":
            rot = _quat_axis_angle(rng.normal(size=3), rng.uniform(-3.0, 3.0))
        elif kind == "rotbig":
            rot = random_rotations(rng, 1)[0]
        ts = 0.005 if kind == "rotbig" else 0.002
        _encode(orc, nodes, i, rng.uniform(-ts, ts, 3).astype(np.float32), rot)
    if kind == "trans" and M >= 40:
        for i, t in zip((5, M // 2, M - 3), ((0.3, -0.2, 0.25), (-0.25, 0.15, -0.2), (0.2, 0.3, -0.3))):
            _encode(orc, nodes, i, np.asarray(t, np.float32))
    return nodes


# ------------------------------------------------------------------ warped-fusion cases -------------------------------------------------------
# id: volume, pose kind, K kind, frame (cols, rows), field kind, M, weight scale, max weight, passes, warp_to_live, expected search path.
# path: 'list' (most runs rank a run candidate list), 'run_overflow' (block lists fit, run lists overflow: tree search), 'block_overflow'
# (block lists overflow: tree search), 'tree' (M < 8: no lists), 'grid' (M > 8192: no BVH, knn8_grid)
CASES = {
    "deep-trans": ("deep", "front", "k2", (637, 471), "trans", 500, 100.0, 64, 2, False, "list"),
    "aniso-rot3-clamps": ("aniso", "tilted", "default", (640, 480), "rot3", 1000, 400.0, 8, 3, False, "list"),
    "rotated-hd": ("rotated", "front", "k2", (1920, 1080), "trans", 500, 0.0, 64, 2, False, "list"),
    "ragged-weights-tiny": ("ragged", "tilted", "default", (7, 5), "weights", 40, 100.0, 8, 3, False, "list"),
    "aniso-inside-m8": ("aniso", "inside", "k2", (640, 480), "identity", 8, 100.0, 64, 2, False, "list"),
    "aniso60-inside": ("aniso60", "inside", "default", (640, 480), "identity", 300, 100.0, 64, 1, False, "list"),
    "deep-m5": ("deep", "front", "default", (640, 480), "trans", 5, 100.0, 64, 3, False, "tree"),
    "lattice": ("lattice", "front", "default", (640, 480), "lattice", 300, 400.0, 8, 3, False, "list"),
    "ragged-grid": ("ragged", "front", "default", (637, 471), "trans", 9000, 100.0, 64, 1, False, "grid"),
    "deep-cluster": ("deep", "front", "default", (640, 480), "cluster", 1200, 100.0, 64, 1, False, "run_overflow"),
    "coarse-spread": ("coarse", "front", "default", (640, 480), "spread", 6000, 100.0, 64, 1, False, "block_overflow"),
    "rotated-w2l": ("rotated", "tilted", "k2", (640, 480), "rot3", 500, 100.0, 64, 2, True, "list"),
    "ragged-rotbig": ("ragged", "front", "k2", (640, 480), "rotbig", 40, 100.0, 64, 1, False, "list"),
    "bench": ("bench", "tilted", "default", (640, 480), "trans", 2000, 100.0, 64, 1, False, "list"),
}


def case(cid):
    vol, pose_kind, kk, (cols, rows), fk, M, ws, maxw, passes, w2l, path = CASES[cid]
    return dict(id=cid, vol=vol, pose=pose_kind, K=frame_K(kk, cols, rows), cols=cols, rows=rows, field=fk, M=M, ws=ws, maxw=maxw,
                passes=passes, w2l=w2l, path=path, dims=VOLUMES[vol][0], vs=voxel_size(vol), trunc=trunc_dist(vol),
                pose_v=f32(volume_pose(vol, pose_kind)), seed=sum(map(ord, cid)))


def case_nodes(orc, c):
    return field(orc, c["field"], c["M"], c["vol"], c["pose"], c["seed"])


def case_depth(c, p):
    return scene_depth(c["vol"], c["pose"], c["cols"], c["rows"], c["K"], p)


def case_world2cam(c, p):
    return world2cam(c["pose"], p, c["w2l"])


def case_vol2cam(c, p):
    """the volume-to-camera map of pass p, in float64 from the float32 poses"""
    W = case_world2cam(c, p)
    R, t = W[0].astype(np.float64), W[1].astype(np.float64)
    return R @ c["pose_v"][0].astype(np.float64), R @ c["pose_v"][1].astype(np.float64) + t

