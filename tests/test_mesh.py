"""CPU checks of the mesh extraction (dfusion.h df_mesh_*): the marching-cubes case table (include/df_mc_table.h) exhaustively, and the
mesh oracle (tests/mesh_oracle.c) on analytic volumes: a sphere gives a closed, consistently wound surface of the right size, an axis-aligned plane
gives exactly two triangles per cube with every vertex on the plane."""
import contextlib
import io
import re
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import mesh_oracle  # noqa: E402
from oracle import orc  # noqa: E402
from scenes import IDENT, pack, sphere_volume  # noqa: E402

CORNERS = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [0, 0, 1], [1, 0, 1], [1, 1, 1], [0, 1, 1]])
EDGES = [(0, 1), (1, 2), (3, 2), (0, 3), (4, 5), (5, 6), (7, 6), (4, 7), (0, 4), (1, 5), (2, 6), (3, 7)]


def _table():
    text = (ROOT / "include" / "df_mc_table.h").read_text()
    body = text[text.index("DF_MC_TRIANGLES_INIT"):]
    rows = [[int(v) for v in r.split(",")] for r in re.findall(r"\{([-0-9, ]+)\}", body)]
    assert len(rows) == 256
    return [[tuple(r[k:k + 3]) for k in range(0, len(r), 3) if r[k] >= 0] for r in rows]


TABLE = _table()


def _inside(case):
    return [(case >> i) & 1 for i in range(8)]


def _on_face(edge, axis, side):
    return all(CORNERS[c][axis] == side for c in EDGES[edge])


def _face_segments(case, axis, side):
    """the undirected triangle edges a case draws on one face of the cube"""
    return {frozenset((t[i], t[(i + 1) % 3])) for t in TABLE[case] for i in range(3)
            if _on_face(t[i], axis, side) and _on_face(t[(i + 1) % 3], axis, side)}


def test_table_matches_its_generator():
    sys.path.insert(0, str(ROOT / "tools"))
    import gen_mc_table
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        gen_mc_table.main()
    assert out.getvalue() == (ROOT / "include" / "df_mc_table.h").read_text()


def test_each_case_uses_exactly_its_sign_changing_edges():
    for case in range(256):
        s = _inside(case)
        changing = {e for e, (a, b) in enumerate(EDGES) if s[a] != s[b]}
        used = {e for t in TABLE[case] for e in t}
        assert used == changing, case
        assert all(len(set(t)) == 3 for t in TABLE[case]), case


def test_inner_triangle_edges_are_shared_by_two_triangles():
    for case in range(256):
        directed = {}
        for t in TABLE[case]:
            for i in range(3):
                directed[(t[i], t[(i + 1) % 3])] = directed.get((t[i], t[(i + 1) % 3]), 0) + 1
        assert all(n == 1 for n in directed.values()), case          # no directed edge twice: consistent winding inside the cube
        for (a, b) in directed:
            on_face = any(_on_face(a, ax, sd) and _on_face(b, ax, sd) for ax in range(3) for sd in (0, 1))
            if on_face:
                assert (b, a) not in directed, (case, a, b)           # a segment on the cube's surface: one triangle
            else:
                assert (b, a) in directed, (case, a, b)               # inside the cube: two triangles, opposite directions


def test_neighbouring_cubes_draw_the_same_segments_on_their_shared_face():
    for axis in range(3):
        # cube B sits one step along `axis` from cube A: A's face at side 1 is B's face at side 0
        corner_map = {}
        for i, c in enumerate(CORNERS):
            if c[axis] == 1:
                d = c.copy(); d[axis] = 0
                corner_map[i] = int(np.flatnonzero((CORNERS == d).all(1))[0])
        edge_sets = [frozenset(e) for e in EDGES]
        edge_map = {e: edge_sets.index(frozenset((corner_map[a], corner_map[b])))
                    for e, (a, b) in enumerate(EDGES) if a in corner_map and b in corner_map}
        for ca in range(256):
            sa = _inside(ca)
            seg_a = {frozenset(edge_map[e] for e in s) for s in _face_segments(ca, axis, 1)}
            for cb in range(256):
                sb = _inside(cb)
                if any(sa[i] != sb[j] for i, j in corner_map.items()):
                    continue
                assert seg_a == _face_segments(cb, axis, 0), (axis, ca, cb)


def test_winding_faces_free_space():
    mid = {e: (CORNERS[a] + CORNERS[b]) / 2 for e, (a, b) in enumerate(EDGES)}
    for case in range(256):
        s = _inside(case)
        for t in TABLE[case]:
            n = np.cross(mid[t[1]] - mid[t[0]], mid[t[2]] - mid[t[0]])
            out = sum((CORNERS[b] - CORNERS[a]) if s[a] else (CORNERS[a] - CORNERS[b]) for a, b in (EDGES[e] for e in t))
            assert n @ out > 0, (case, t)                              # right-hand normal towards the F > 0 corners


# ------------------------------------------------------------------ oracle on analytic volumes --------------------------------------------
def mesh_of(vol, dims, vsz, trunc):
    cloud = orc.extract_cloud(vol, dims, vsz, trunc, 64, IDENT, int(np.prod(dims)) * 3)
    tris = mesh_oracle.mesh(vol, dims, len(cloud))
    assert tris is not None
    return cloud[:, :3].astype(np.float64), tris


def test_vertex_map_numbers_the_cloud():
    vol, dims, vsz, trunc, _, _ = sphere_volume()
    cloud = orc.extract_cloud(vol, dims, vsz, trunc, 64, IDENT, int(np.prod(dims)) * 3)
    m = mesh_oracle.vertex_map(vol, dims)
    z, y, x, axis = np.nonzero(m >= 0)
    idx = m[z, y, x, axis]
    assert np.array_equal(np.sort(idx), np.arange(len(cloud)))
    vs = np.float32(vsz[0])
    centre = np.stack([(x + np.float32(0.5)) * vs, (y + np.float32(0.5)) * vs, (z + np.float32(0.5)) * vs], 1).astype(np.float32)
    p = cloud[idx, :3]
    for a in range(3):                                                   # on the voxel's edge along `axis`: the other two coordinates exact
        off = axis != a
        assert np.array_equal(p[off, a], centre[off, a])
        on = axis == a
        assert np.all((p[on, a] >= centre[on, a]) & (p[on, a] <= centre[on, a] + vs))


def test_sphere_is_a_closed_surface_of_the_right_size():
    vol, dims, vsz, trunc, c, R = sphere_volume()
    v, tris = mesh_of(vol, dims, vsz, trunc)
    assert len(tris) > 5000
    e = np.sort(np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]]), 1)
    _, counts = np.unique(e, axis=0, return_counts=True)
    assert counts.min() == 2 and counts.max() == 2                       # no boundary edge, no edge of three faces
    directed = np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]])
    assert len(np.unique(directed, axis=0)) == len(directed)             # each edge once in each direction: consistent winding
    used = np.unique(tris)
    assert len(used) - len(counts) + len(tris) == 2                       # V - E + F of a sphere
    r = np.linalg.norm(v[used] - c, axis=1)
    assert np.abs(r - R).max() < vsz[0] / 10
    a, b, cc = v[tris[:, 0]], v[tris[:, 1]], v[tris[:, 2]]
    n = np.cross(b - a, cc - a)
    big = np.linalg.norm(n, axis=1) > 1e-12
    assert np.all(np.einsum("ij,ij->i", n[big], (a + b + cc)[big] / 3 - c) > 0)   # normals point away from the centre (F > 0 outside)
    vol_signed = np.einsum("ij,ij->i", a - c, np.cross(b - c, cc - c)).sum() / 6
    assert abs(vol_signed / (4 / 3 * np.pi * R ** 3) - 1) < 0.01


def test_plane_at_a_fractional_offset():
    dims, vs = (20, 12, 10), 0.02
    Dx, Dy, Dz = dims
    z0 = (4.3 + 0.5) * vs                                                # between the centres of slices 4 and 5
    z = np.arange(Dz)[:, None, None] * np.ones((1, Dy, Dx))
    F = np.clip(((z + 0.5) * vs - z0) / (3 * vs), -1.0, 1.0)
    vol = pack(F)
    v, tris = mesh_of(vol, dims, (vs, vs, vs), 3 * vs)
    assert len(tris) == 2 * (Dx - 1) * (Dy - 1)
    pz = v[np.unique(tris), 2].astype(np.float32)
    assert np.all(pz.view(np.uint32) == pz[0].view(np.uint32))          # every vertex on one plane, bit for bit
    assert abs(pz[0] - z0) < 1e-3 * vs
    n = np.cross(v[tris[:, 1]] - v[tris[:, 0]], v[tris[:, 2]] - v[tris[:, 0]])
    assert np.all(n[:, 2] > 0) and np.allclose(n[:, :2], 0)             # facing +z, where F > 0


def test_a_cloud_of_another_size_is_refused():
    vol, dims, vsz, trunc, _, _ = sphere_volume()
    cloud = orc.extract_cloud(vol, dims, vsz, trunc, 64, IDENT, int(np.prod(dims)) * 3)
    assert mesh_oracle.mesh(vol, dims, len(cloud) - 1) is None


def test_save_ply_with_faces(tmp_path):
    from dynamicfusion_b200 import host
    pts = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [np.nan, 0, 0]], np.float32)
    nrm = np.array([[0, 0, 1], [0, 0, 1], [np.nan, 0, 1], [0, 0, 1]], np.float32)
    faces = np.array([[0, 1, 2]], np.int32)
    path = tmp_path / "m.ply"
    assert host.save_ply(path, pts, nrm, faces) == 4                     # every vertex kept: indices stay valid
    data = path.read_bytes()
    head = data[:data.index(b"end_header\n") + len(b"end_header\n")]
    assert head == (b"ply\nformat binary_little_endian 1.0\ncomment dynamicfusion mesh\nelement vertex 4\nproperty float x\n"
                    b"property float y\nproperty float z\nproperty float nx\nproperty float ny\nproperty float nz\nelement face 1\n"
                    b"property list uchar int vertex_indices\nend_header\n")
    body = data[len(head):]
    v = np.frombuffer(body[:4 * 24], "<f4").reshape(4, 6)
    assert np.array_equal(v[:3, :3], pts[:3]) and np.isnan(v[3, 0]) and np.array_equal(v[2, 3:], [0, 0, 0])
    assert body[4 * 24] == 3 and np.array_equal(np.frombuffer(body[4 * 24 + 1:], "<i4"), [0, 1, 2])
    with pytest.raises(ValueError):
        host.save_ply(path, pts, nrm, np.array([[0, 1, 4]]))


def test_save_ply_without_faces_is_unchanged(tmp_path):
    from dynamicfusion_b200 import host
    pts = np.array([[0, 0, 0], [np.nan, 0, 0], [1, 2, 3]], np.float32)
    path = tmp_path / "c.ply"
    assert host.save_ply(path, pts) == 2
    assert path.read_bytes() == (b"ply\nformat binary_little_endian 1.0\ncomment dynamicfusion canonical cloud\nelement vertex 2\n"
                                 b"property float x\nproperty float y\nproperty float z\nend_header\n" + pts[[0, 2]].astype("<f4").tobytes())
