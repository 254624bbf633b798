"""CPU checks of df_mesh_correspond's rule (dfusion.h) through its C oracle (tests/correspond_oracle.c), run on rasterisations by the raster
oracle: a source mesh that is a rigid motion of the drawn one gives the moved drawn points, the barycentric weights are a partition of unity
inside the triangle, the drawn mesh as its own source gives the drawn points back with camera-facing normals, and every no-correspondence
case writes NaNs."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import color_oracle  # noqa: E402
import correspond_oracle as co  # noqa: E402
import raster_oracle  # noqa: E402
from scenes import IDENT, K_EXACT, SPHERE_COLS, SPHERE_K, SPHERE_ROWS, look_at, plane_verts, sphere_mesh  # noqa: E402


def _rot(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def _moved(verts, R, t):
    out = np.array(verts, np.float32, copy=True)
    out[:, :3] = (verts[:, :3].astype(np.float64) @ R.T + t).astype(np.float32)
    return out


def _quad():
    verts = plane_verts([(2, 2), (10, 2), (10, 8), (2, 8)])
    return verts, np.array([[0, 2, 1], [0, 3, 2]], np.int32), IDENT, K_EXACT, 16, 12


def _sphere():
    cloud, tris, centre, _, _ = sphere_mesh()
    return cloud, tris, look_at(centre, 0.6, (0.3, -0.2, 1.0)), SPHERE_K, SPHERE_COLS, SPHERE_ROWS


def _cam_to_world(P, w2c):
    R, t = (np.asarray(a, np.float64) for a in w2c)
    return (P[..., :3].astype(np.float64) - t) @ R                  # R^T (P - t)


def test_rigidly_moved_source_gives_the_moved_drawn_points():
    R, t = _rot(0.3, -0.2, 0.5), np.array([0.05, -0.02, 0.1])
    for name, (verts, tris, w2c, K, cols, rows) in (("quad", _quad()), ("sphere", _sphere())):
        ids, pts, _, _ = raster_oracle.raster(verts, tris, w2c, K, cols, rows)
        drawn = ids >= 0
        assert drawn.sum() > 40, name
        src = _moved(verts, R, t)
        sp, sn = co.correspond(ids, pts, verts, src, tris, w2c)
        want = _cam_to_world(pts, w2c) @ R.T + t
        assert np.all(np.isnan(sp[~drawn])) and np.all(np.isnan(sn[~drawn]))
        assert np.all(sp[drawn][:, 3] == 0) and np.all(sn[drawn][:, 3] == 0)
        err = np.abs(sp[drawn][:, :3] - want[drawn])
        scale = np.abs(want[drawn]).max()
        assert err.max() <= 4e-6 * max(scale, 1.0), (name, err.max())
        # the source normal is the moved face normal of the drawn triangle (float32 cross products of the mesh's slivers round at 1e-5)
        assert np.allclose(sn[drawn][:, :3], _face_normals(verts, tris, ids[drawn]) @ R.T, atol=1e-4), name
        assert np.allclose(np.linalg.norm(sn[drawn][:, :3].astype(np.float64), axis=1), 1.0, atol=1e-6)


def _face_normals(verts, tris, ids):
    """unit face normals cross(v1 - v0, v2 - v0) of triangles `ids`, float64"""
    v = verts[:, :3].astype(np.float64)
    f = tris[ids]
    n = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    return n / np.linalg.norm(n, axis=1, keepdims=True)


def test_weights_are_a_partition_of_unity_inside_the_triangle():
    for name, (verts, tris, w2c, K, cols, rows) in (("quad", _quad()), ("sphere", _sphere())):
        ids, pts, _, _ = raster_oracle.raster(verts, tris, w2c, K, cols, rows)
        drawn = ids >= 0
        b = co.weights(ids, pts, verts, tris, w2c)
        assert np.all(np.isnan(b[~drawn]))
        bd = b[drawn].astype(np.float64)
        assert np.all(np.isfinite(bd)), name
        assert np.abs(bd.sum(1) - 1.0).max() <= 1e-6, name
        # the sample lies inside the SNAPPED triangle; the rule's weights are those of the unsnapped one.  A corner moves by at most
        # sqrt(2)/512 px when snapped, which moves a weight by at most that times |grad b| (px^-1) per corner: exact geometry (the quad)
        # gives no slack
        slack = 3 * np.sqrt(2) / 512 * _max_weight_gradient(verts, tris, w2c, K, ids[drawn])
        assert np.all(bd.min(1) >= -1e-5 - slack) and np.all(bd.max(1) <= 1 + 1e-5 + slack), name
        if name == "quad":
            assert bd.min() >= -1e-5 and bd.max() <= 1 + 1e-5


def _max_weight_gradient(verts, tris, w2c, K, ids):
    """per triangle of `ids`: the largest |grad b_k| over its corners in the image (px^-1) = longest edge / (2 area)"""
    R, t = (np.asarray(a, np.float64) for a in w2c)
    c = verts[:, :3].astype(np.float64) @ R.T + t
    uv = np.stack([K[0] * c[:, 0] / c[:, 2] + K[2], K[1] * c[:, 1] / c[:, 2] + K[3]], 1)
    f = tris[ids]
    a, b, d = uv[f[:, 0]], uv[f[:, 1]], uv[f[:, 2]]
    area2 = np.abs((b[:, 0] - a[:, 0]) * (d[:, 1] - a[:, 1]) - (b[:, 1] - a[:, 1]) * (d[:, 0] - a[:, 0]))
    longest = np.max([np.linalg.norm(b - a, axis=1), np.linalg.norm(d - b, axis=1), np.linalg.norm(a - d, axis=1)], 0)
    return longest / area2


def test_the_drawn_mesh_as_its_own_source_gives_the_drawn_points():
    verts, tris, w2c, K, cols, rows = _sphere()
    cam = _moved(verts, np.asarray(w2c[0], np.float64), np.asarray(w2c[1], np.float64))   # the mesh in the camera frame: drawn at IDENT
    for v, T, K_, c, r in ((cam, tris, K, cols, rows), _quad()[:2] + _quad()[3:]):
        ids, pts, nrm, _ = raster_oracle.raster(v, T, IDENT, K_, c, r)
        drawn = ids >= 0
        sp, sn = co.correspond(ids, pts, v, v, T, IDENT)
        d = np.abs(sp[drawn][:, :3] - pts[drawn][:, :3])
        assert d.max() <= 4e-6 * np.abs(pts[drawn][:, :3]).max()
        assert np.all(np.einsum("ij,ij->i", sn[drawn][:, :3], pts[drawn][:, :3]) < 0)     # facing the camera
        assert np.allclose(sn[drawn], nrm[drawn], atol=1e-6)         # the raster's normal, up to the rounding of the camera transform


def test_no_correspondence_cases_write_nans():
    verts, tris, w2c, K, cols, rows = _quad()
    ids, pts, _, _ = raster_oracle.raster(verts, tris, w2c, K, cols, rows)
    drawn = ids >= 0
    sp, _ = co.correspond(ids, pts, verts, verts, tris, w2c)
    assert np.all(np.isnan(sp[ids == -1])) and np.all(~np.isnan(sp[drawn]))
    j, i = np.argwhere(drawn)[7]
    # den zero (the pixel's triangle has all three corners on one vertex) and den not finite (a corner at 1e30)
    bad_ids = ids.copy()
    deg = np.concatenate([tris, [[0, 0, 0], [0, 1, 4]]]).astype(np.int32)
    far = np.concatenate([verts, [[1e30, 0.0, 1.0]]]).astype(np.float32)
    for t in (2, 3):
        bad_ids[j, i] = t
        sp, sn = co.correspond(bad_ids, pts, far, far, deg, w2c)
        assert np.all(np.isnan(sp[j, i])) and np.all(np.isnan(sn[j, i])), t
        assert np.all(~np.isnan(sp[drawn & (bad_ids != t)]))
    # the target map: NaN vertex, and the distance gate on both sides of max_dist
    target = pts.copy()
    target[..., 0] += np.float32(0.15)
    target[..., 2] += np.float32(0.2)                                   # |T - P| = 0.25
    target[j, i] = np.nan
    near, _ = co.correspond(ids, pts, verts, verts, tris, w2c, target, 0.251)
    assert np.all(np.isnan(near[j, i]))
    keep = drawn.copy(); keep[j, i] = False
    assert np.all(~np.isnan(near[keep]))
    far_, _ = co.correspond(ids, pts, verts, verts, tris, w2c, target, 0.249)
    assert np.all(np.isnan(far_))
    free, _ = co.correspond(ids, pts, verts, verts, tris, w2c)
    assert np.array_equal(near[keep].view(np.uint32), free[keep].view(np.uint32))   # the distance test changes nothing else


def test_host_affine_helpers_match_numpy():
    A = (_rot(0.1, 0.2, -0.3).astype(np.float32), np.array([0.1, -0.2, 0.3], np.float32))
    B = (_rot(-0.2, 0.05, 0.4).astype(np.float32), np.array([-0.05, 0.02, 0.7], np.float32))
    R, t = color_oracle.aff_mul(A, B)
    assert np.allclose(R, A[0].astype(np.float64) @ B[0], atol=1e-6) and np.allclose(t, A[0].astype(np.float64) @ B[1] + A[1], atol=1e-6)
    Ri, ti = color_oracle.aff_inv(A)
    assert np.allclose(Ri @ A[0], np.eye(3), atol=1e-6) and np.allclose(Ri @ A[1] + ti, 0, atol=1e-6)
