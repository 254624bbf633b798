"""CPU checks of the rasteriser's rule (dfusion.h df_raster_mesh) through its C oracle (tests/raster_oracle.c): the top-left rule and
watertight shared edges on exact pixel-centre geometry, exact single coverage of an analytic sphere's marching-cubes mesh away from its
silhouette, drawn points on the sphere, the skip and tie rules, and the geometry of the output maps."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import raster_oracle  # noqa: E402
from scenes import IDENT, K_EXACT, SPHERE_COLS, SPHERE_K, SPHERE_ROWS, look_at, plane_verts, sphere_mesh  # noqa: E402


def test_quad_sharing_a_diagonal_is_covered_once_with_top_left_edges():
    verts = plane_verts([(2, 2), (10, 2), (10, 8), (2, 8)])
    tris = np.array([[0, 2, 1], [0, 3, 2]], np.int32)            # camera-facing: negative fixed-point area, the diagonal 0-2 in both
    cov = raster_oracle.coverage(verts, tris, IDENT, K_EXACT, 16, 12)
    want = np.zeros((12, 16), np.int32)
    want[2:8, 2:10] = 1                                            # top row j = 2 and left column i = 2 in; bottom j = 8, right i = 10 out
    assert np.array_equal(cov, want)
    assert cov[5, 6] == 1                                          # (6, 5) lies on the diagonal
    ids, _, _, stats = raster_oracle.raster(verts, tris, IDENT, K_EXACT, 16, 12)
    assert int((ids >= 0).sum()) == 48 and stats[4] == 48
    assert stats[0] == 0 and stats[1] == 0 and stats[2] + stats[3] == 2
    # which side of the diagonal: below-left is triangle 1, above-right triangle 0
    assert ids[7, 2] == 1 and ids[2, 9] == 0


def test_fan_around_a_pixel_centre_covers_it_once():
    c = np.array([20.0, 20.0])
    ring = [c + np.array([5 * np.cos(a), 5 * np.sin(a)]) for a in np.arange(8) * np.pi / 4]
    ring = [np.round(r * 2) / 2 for r in ring]                     # half-pixel positions, exact in 8 sub-pixel bits
    verts = plane_verts([c] + ring)
    tris = np.array([[0, 1 + (k + 1) % 8, 1 + k] for k in range(8)], np.int32)
    cov = raster_oracle.coverage(verts, tris, IDENT, K_EXACT, 40, 40)
    assert cov[20, 20] == 1
    assert cov.max() == 1
    assert np.all(cov[16:25, 16:25][np.hypot(*np.mgrid[-4:5, -4:5]) < 3.5] == 1)


def test_reversed_winding_draws_nothing():
    verts = plane_verts([(2, 2), (10, 2), (10, 8), (2, 8)])
    tris = np.array([[0, 1, 2], [0, 2, 3]], np.int32)
    ids, pts, nrm, stats = raster_oracle.raster(verts, tris, IDENT, K_EXACT, 16, 12)
    assert np.all(ids == -1) and np.all(np.isnan(pts)) and np.all(np.isnan(nrm))
    assert list(stats) == [2, 0, 0, 0, 0]
    assert raster_oracle.coverage(verts, tris, IDENT, K_EXACT, 16, 12).max() == 0


def test_skipped_triangles_are_counted():
    good = plane_verts([(2, 2), (10, 2), (10, 8)])
    near = good.copy(); near[1, 2] = 0.005                         # c.z < DF_RASTER_NEAR
    guard = good.copy(); guard[1, 0] = 3000.0                      # u = 96000 px: outside the +-2^16 band
    nonfinite = good.copy(); nonfinite[2, 1] = np.inf
    for verts in (near, guard, nonfinite):
        ids, _, _, stats = raster_oracle.raster(verts, [[0, 2, 1]], IDENT, K_EXACT, 16, 12)
        assert list(stats) == [0, 1, 0, 0, 0] and np.all(ids == -1)
    for bad in ([0, 3, 1], [0, -1, 1], [2**31 - 1, 2, 1]):
        ids, _, _, stats = raster_oracle.raster(good, [bad], IDENT, K_EXACT, 16, 12)
        assert list(stats) == [0, 1, 0, 0, 0] and np.all(ids == -1)
    ids, _, _, stats = raster_oracle.raster(good, [[0, 2, 1]], IDENT, K_EXACT, 16, 12)
    assert stats[1] == 0 and stats[4] > 0


def test_identical_triangles_the_smaller_index_wins():
    verts = plane_verts([(2, 2), (10, 2), (10, 8)])
    ids, _, _, stats = raster_oracle.raster(verts, [[0, 2, 1]] * 3, IDENT, K_EXACT, 16, 12)
    drawn = ids >= 0
    assert drawn.sum() > 10 and np.all(ids[drawn] == 0)
    assert stats[2] + stats[3] == 3
    # a nearer copy with a larger index wins over a farther one with a smaller index
    far = verts * np.float32(2.0)                                  # the same image triangle at twice the depth
    both = np.concatenate([far, verts])
    ids, pts, _, _ = raster_oracle.raster(both, [[0, 2, 1], [3, 5, 4]], IDENT, K_EXACT, 16, 12)
    assert np.all(ids[ids >= 0] == 1) and np.allclose(pts[ids >= 0][:, 2], 1.0)


# ------------------------------------------------------------------ the analytic sphere ------------------------------------------------------
def _ray_dirs(K, cols, rows):
    fx, fy, cx, cy = (np.float32(v) for v in K)
    i = np.arange(cols, dtype=np.float32)[None, :]
    j = np.arange(rows, dtype=np.float32)[:, None]
    dx = (i - cx) * (np.float32(1) / fx)
    dy = (j - cy) * (np.float32(1) / fy)
    return np.broadcast_to(dx, (rows, cols)), np.broadcast_to(dy, (rows, cols))


def test_sphere_is_covered_once_inside_its_silhouette_and_drawn_on_it():
    cloud, tris, centre, radius, vs = sphere_mesh()
    R, t = look_at(centre, 0.8)
    cov = raster_oracle.coverage(cloud, tris, (R, t), SPHERE_K, SPHERE_COLS, SPHERE_ROWS)
    dx, dy = _ray_dirs(SPHERE_K, SPHERE_COLS, SPHERE_ROWS)
    d = np.stack([dx, dy, np.ones_like(dx)], -1).astype(np.float64)
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    cc = R.astype(np.float64) @ centre + t                         # the centre in the camera frame
    miss = np.linalg.norm(cc - (d @ cc)[..., None] * d, axis=-1)   # distance of each pixel's ray from the centre
    inside, outside = miss < radius - 1.5 * vs, miss > radius + 1.5 * vs
    assert inside.sum() > 2000 and outside.sum() > 2000
    assert np.all(cov[inside] == 1)
    assert np.all(cov[outside] == 0)
    ids, pts, nrm, stats = raster_oracle.raster(cloud, tris, (R, t), SPHERE_K, SPHERE_COLS, SPHERE_ROWS)
    drawn = ids >= 0
    assert np.all(drawn[inside]) and not np.any(drawn[outside])
    r = np.linalg.norm(pts[drawn][:, :3].astype(np.float64) - cc, axis=-1)
    assert np.abs(r - radius).max() <= 0.25 * vs                   # vs/10 vertex bound plus chord sag
    assert stats[4] == drawn.sum() and stats[0] > 0 and stats[1] == 0


def test_output_geometry():
    cloud, tris, centre, _, _ = sphere_mesh()
    R, t = look_at(centre, 0.6, (0.3, -0.2, 1.0))
    ids, pts, nrm, _ = raster_oracle.raster(cloud, tris, (R, t), SPHERE_K, SPHERE_COLS, SPHERE_ROWS)
    drawn = ids >= 0
    assert drawn.sum() > 3000
    assert np.all(np.isnan(pts[~drawn])) and np.all(np.isnan(nrm[~drawn]))
    n, p = nrm[drawn], pts[drawn]
    assert np.all(n[:, 3] == 0) and np.all(p[:, 3] == 0)
    assert np.allclose(np.linalg.norm(n[:, :3].astype(np.float64), axis=1), 1.0, atol=1e-6)
    assert np.all(np.einsum("ij,ij->i", n[:, :3], p[:, :3]) < 0)  # facing the camera
    dx, dy = _ray_dirs(SPHERE_K, SPHERE_COLS, SPHERE_ROWS)
    assert np.array_equal(p[:, 0], dx[drawn] * p[:, 2]) and np.array_equal(p[:, 1], dy[drawn] * p[:, 2])   # on the pixel's ray, bit for bit
    assert np.all(p[:, 2] > 0)
