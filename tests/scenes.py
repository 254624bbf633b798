"""CPU scenes the tests share: the analytic sphere's volume and marching-cubes mesh, cameras that look at it, pixel-exact plane triangles,
the colour tests' small scene, and the data-term solve's node patch.  Test infrastructure only."""
import numpy as np

import mesh_oracle
from oracle import orc

IDENT = (np.eye(3, dtype=np.float32), np.zeros(3, np.float32))

# pixel-exact camera: u = fma(32, x / 1, 0) is an integer for x = i / 32 on the plane z = 1
K_EXACT = (32.0, 32.0, 0.0, 0.0)
SPHERE_K = (150.0, 150.0, 79.5, 59.5)
SPHERE_COLS, SPHERE_ROWS = 160, 120
K640 = (525.0, 525.0, 319.5, 239.5)


def pack(F, W=1):
    return (np.asarray(F, np.float16).view(np.uint16).astype(np.uint32) | (np.uint32(W) << np.uint32(16))).ravel()


def sphere_volume(dims=(64, 60, 56), vs=0.01, radius_vox=20.3, centre_vox=(31.6, 29.8, 27.3), trunc_vox=4.0):
    Dx, Dy, Dz = dims
    z, y, x = np.meshgrid(np.arange(Dz), np.arange(Dy), np.arange(Dx), indexing="ij")
    c = np.asarray(centre_vox) * vs
    d = np.sqrt(((x + 0.5) * vs - c[0]) ** 2 + ((y + 0.5) * vs - c[1]) ** 2 + ((z + 0.5) * vs - c[2]) ** 2) - radius_vox * vs
    F = np.clip(d / (trunc_vox * vs), -1.0, 1.0)
    return pack(F), dims, (vs, vs, vs), trunc_vox * vs, c, radius_vox * vs


def sphere_mesh():
    """the marching-cubes mesh of sphere_volume (float32 [N, 4] cloud, int32 [T, 3]), its centre and radius (m), voxel size"""
    vol, dims, vsz, trunc, centre, radius = sphere_volume()
    cloud = orc.extract_cloud(vol, dims, vsz, trunc, 64, IDENT, int(np.prod(dims)) * 3)
    tris = mesh_oracle.mesh(vol, dims, len(cloud))
    return np.ascontiguousarray(cloud, np.float32), tris, np.asarray(centre, np.float64), float(radius), float(vsz[0])


def look_at(centre, distance, direction=(0.0, 0.0, 1.0)):
    """world-to-camera (R, t) of a camera `distance` from `centre` looking along `direction` (camera y roughly down the world's y)"""
    f = np.asarray(direction, np.float64); f /= np.linalg.norm(f)
    up = np.array([0.0, 1.0, 0.0]) if abs(f[1]) < 0.9 else np.array([1.0, 0.0, 0.0])
    x = np.cross(up, f); x /= np.linalg.norm(x)
    y = np.cross(f, x)
    R = np.stack([x, y, f])                                        # rows: camera axes in world coordinates
    eye = np.asarray(centre, np.float64) - distance * f
    return R.astype(np.float32), (-R @ eye).astype(np.float32)


def plane_verts(uv):
    """vertices on the plane z = 1 that K_EXACT projects to the pixel positions uv"""
    uv = np.asarray(uv, np.float64)
    return np.stack([uv[:, 0] / 32.0, uv[:, 1] / 32.0, np.ones(len(uv))], 1).astype(np.float32)


# ------------------------------------------------------------------------------------------------------------ the colour tests' scene
DIMS = (32, 24, 20)
VS = (0.02, 0.02, 0.02)
TRUNC = 0.06
BAND = 0.5 * TRUNC
COLS, ROWS = 64, 48
K = (60.0, 60.0, 32.0, 24.0)
VOL2CAM = (np.eye(3, dtype=np.float32), np.array([-0.32, -0.24, 0.5], np.float32))
PLANE_Z = 0.7


def plane_dists(z=PLANE_Z):
    u, v = np.meshgrid(np.arange(COLS, dtype=np.float64), np.arange(ROWS, dtype=np.float64))
    ray = np.sqrt(((u - K[2]) / K[0]) ** 2 + ((v - K[3]) / K[1]) ** 2 + 1.0)
    return (z * ray).astype(np.float16).view(np.uint16)


def constant_image(bgr):
    img = np.empty((ROWS, COLS, 4), np.uint8)
    img[..., :3] = bgr
    img[..., 3] = 255
    return img


def word(r, g, b, w):
    return r | (g << 8) | (b << 16) | (w << 24)


# ------------------------------------------------------------------------------------------------------------- the data-term solve's patch
def node_patch(rng, n=2500):
    """a 10 x 6 node grid on the plane z = 1 and n source points on a gently curved patch over it"""
    gx, gy = np.meshgrid(np.linspace(-0.3, 0.3, 10), np.linspace(-0.2, 0.2, 6))
    node_pts = np.stack([gx.ravel(), gy.ravel(), np.full(gx.size, 1.0)], 1).astype(np.float32)
    src = np.zeros((n, 4), np.float32)
    src[:, 0] = rng.uniform(-0.3, 0.3, n); src[:, 1] = rng.uniform(-0.2, 0.2, n); src[:, 2] = 1.0 + 0.02 * np.sin(8 * src[:, 0])
    return node_pts, src


def rot_y(deg):
    a = np.deg2rad(deg)
    return np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
