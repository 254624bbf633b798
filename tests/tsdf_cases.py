"""Shapes of the TSDF stage's float64 tests: non-cubic volumes on both sides of every integrate dispatch, anisotropic voxels, ragged and
pitched frames, intrinsics with fx != fy and an off-centre principal point, and the camera poses.  CPU only (numpy and synth)."""
from __future__ import annotations

import numpy as np

from dynamicfusion_b200 import synth

DEFAULT_K = tuple(float(k) for k in synth.DEFAULT_K)
K2 = (585.0, 548.5, 331.75, 226.25)              # fx != fy, principal point off the image centre
TRUNC = 0.04
MAX_W = 64
STEP_FACTOR = 0.75
DELTA_FACTOR = 0.5

# name: (dims, size in metres); the comment says what the shape exercises
VOLUMES = {
    "v5_iso": ((128, 64, 96), (1.0, 0.5, 0.75)),          # packed kernel, isotropic voxels, non-cubic
    "v5_aniso": ((96, 80, 80), (1.2, 0.8, 0.6)),          # packed kernel, three voxel sizes, last z-chunk 16 of 32
    "v5_deep": ((96, 48, 300), (0.96, 0.48, 1.5)),        # Dz >= 256: z-chunk 64, last one 44
    "plain4": ((64, 72, 130), (0.64, 0.72, 1.04)),        # Dy % 16 != 0: integrate_kernel<4>, last z-chunk 2 of 32
    "plain1": ((30, 34, 38), (0.6, 0.51, 0.76)),          # Dx % 4 != 0: integrate_kernel<1>, anisotropic
    "ragged": ((32, 44, 37), (0.4, 0.55, 0.37)),          # 52,096 voxels: neither 1024-voxel stretches nor 8^3 bricks divide it
}

FRAMES = [(640, 480), (641, 479), (320, 240), (1920, 1080), (7, 5)]
PITCH_PAD = [0, 2, 512]                                    # bytes added to each row of the depth and distance images


def voxel_size(name):
    dims, size = VOLUMES[name]
    return (np.asarray(size, np.float32) / np.asarray(dims, np.float32)).astype(np.float32)


def trunc_dist(name):
    """TsdfVolume::setTruncDist's rule: at least 2.1 voxels of the largest voxel size"""
    return float(max(np.float32(TRUNC), np.float32(2.1) * voxel_size(name).max()))


def _aff(R, t):
    return np.asarray(R, np.float64), np.asarray(t, np.float64)


def _mul(A, B):
    return A[0] @ B[0], A[0] @ B[1] + A[1]


def _inv(A):
    Ri = A[0].T
    return Ri, -Ri @ A[1]


def f32(A):
    return np.ascontiguousarray(A[0], np.float32), np.ascontiguousarray(A[1], np.float32)


def _rot(ax, deg):
    a = np.deg2rad(deg)
    c, s = np.cos(a), np.sin(a)
    if ax == "x":
        return np.array([[1, 0, 0], [0, c, -s], [0, s, c]])
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def volume_pose(name, pose_kind):
    """volume-to-world: the volume about the optical axis, its near face 0.5 m in front of the camera; for 'inside' the camera plane cuts
    the volume at 30 % of its depth.  The offsets of a millimetre or two keep voxel centres off the planes x = 0 and y = 0, where a
    principal point on a whole pixel would put whole slices of voxels exactly on a pixel edge (ties the float32 chain decides either way)."""
    size = VOLUMES[name][1]
    z0 = -0.3 * size[2] if pose_kind == "inside" else 0.5
    return _aff(np.eye(3), (-size[0] / 2 + 0.00137, -size[1] / 2 - 0.00091, z0 + 0.00213))


def camera_pose(name, pose_kind):
    """camera-to-world of the integration (front, tilted, inside: the camera at the origin) or of the ray-cast from behind the surface"""
    size = np.asarray(VOLUMES[name][1])
    if pose_kind in ("front", "inside"):
        return _aff(np.eye(3), np.zeros(3))
    if pose_kind == "tilted":
        return _aff(_rot("x", 7.0) @ _rot("y", -4.0), (0.03, -0.02, 0.05))
    assert pose_kind == "behind"
    centre = np.array([0.0, 0.0, 0.5 + size[2] / 2])
    R = _rot("y", 125.0) @ _rot("x", 8.0)                 # looks back towards the camera side, obliquely
    return _aff(R, centre - R @ np.array([0.0, 0.0, 0.7 * size.max() + 0.3]))


def scene_depth(name, pose_kind, cols, rows, K, frame):
    """u16 depth of a sphere in front of a wall, both inside the volume's depth range (noise and dropout differ per frame)"""
    size = VOLUMES[name][1]
    lo = volume_pose(name, pose_kind)[1][2]
    lo = max(lo, 0.08)
    hi = volume_pose(name, pose_kind)[1][2] + size[2]
    r = 0.3 * min(size[0], size[1], hi - lo)
    return synth.sphere_wall_depth(cols=cols, rows=rows, K=K, seed=1000 * frame + cols, radius=r, centre=(0.02, -0.01, lo + 0.45 * (hi - lo)),
                                   wall_z=lo + 0.85 * (hi - lo))


def frame_pose(name, pose_kind, frame):
    """camera-to-world of frame 0, 1, 2: the case's pose, then small moves (the running average sees different samples)"""
    P = camera_pose(name, pose_kind)
    moves = [_aff(np.eye(3), np.zeros(3)), _aff(np.eye(3), (0.004, 0.0, 0.002)), _aff(_rot("y", 0.4), (-0.003, 0.002, 0.0))]
    return _mul(P, moves[frame])


def vol2cam(name, pose_kind, frame):
    return f32(_mul(_inv(frame_pose(name, pose_kind, frame)), volume_pose(name, pose_kind)))


def cam2vol(name, pose_kind, view):
    return f32(_mul(_inv(volume_pose(name, pose_kind)), camera_pose(name, view)))


def frame_K(cols, rows, K=K2):
    """K scaled from 640 x 480 to the frame"""
    return (K[0] * cols / 640.0, K[1] * rows / 480.0, K[2] * cols / 640.0, K[3] * rows / 480.0)


# (volume, integration pose, K, ray-cast view) at 640 x 480: every volume at two pose / K pairs
VOLUME_CASES = [
    ("v5_iso", "front", DEFAULT_K, "front"), ("v5_iso", "tilted", K2, "behind"),
    ("v5_aniso", "tilted", DEFAULT_K, "tilted"), ("v5_aniso", "inside", K2, "inside"),
    ("v5_deep", "front", K2, "front"), ("v5_deep", "tilted", DEFAULT_K, "behind"),
    ("plain4", "front", DEFAULT_K, "front"), ("plain4", "inside", K2, "behind"),
    ("plain1", "tilted", K2, "tilted"), ("plain1", "front", DEFAULT_K, "behind"),
    ("ragged", "front", K2, "front"), ("ragged", "tilted", DEFAULT_K, "behind"),
]

# (volume, frame size): every frame size on one packed-kernel and one plain-kernel volume, each at every pitch
FRAME_CASES = [(v, f) for v in ("v5_iso", "plain4") for f in FRAMES]
