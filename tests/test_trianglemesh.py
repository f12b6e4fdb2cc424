"""Mesh extraction without a GPU: the generated marching-cubes table (oracle/mc_table.py -> csrc/mc_table.cuh), the float64 whole-volume
restatement of the kernels (oracle/mesh.py) on analytic volumes, and the PLY writer of neuralsim_b200/graphics/trianglemesh.py."""
import os

import numpy as np
import pytest

from oracle import mc_table
from oracle import mesh as omesh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ the case table
def test_committed_table_is_the_generators_output():
    with open(os.path.join(ROOT, "neuralsim_b200", "csrc", "mc_table.cuh")) as f:
        assert f.read() == mc_table.render_cuh()


def test_empty_cases_and_count_bound():
    count, edges = mc_table.build_table()
    assert count[0] == 0 and count[255] == 0
    assert count.max() == mc_table.MAX_TRIS == 5
    for c in range(256):
        assert (edges[c, 3 * count[c]:] == -1).all() and (edges[c, :3 * count[c]] >= 0).all()


def test_vertices_are_the_crossing_edges_and_complement_keeps_them():
    for c in range(256):
        used = sorted(set(e for t in mc_table.case_triangles(c) for e in t))
        assert used == mc_table.crossing_edges(c), c
        assert mc_table.crossing_edges(c) == mc_table.crossing_edges(255 - c), c


def _face_of(e0, e1):
    """(axis, side) of the cube face holding both edges, or None"""
    pts = [set(map(tuple, mc_table.CORNER[list(mc_table.EDGE_CORNERS[e])])) for e in (e0, e1)]
    for a in range(3):
        for s in range(2):
            if all(all(p[a] == s for p in ps) for ps in pts):
                return a, s
    return None


def test_mesh_edges_on_each_face_are_the_face_rule_segments():
    for c in range(256):
        on_face = {}
        for t in mc_table.case_triangles(c):
            for u, v in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0])):
                f = _face_of(u, v)
                if f is not None:
                    on_face.setdefault(f, []).append(frozenset((u, v)))
        for a in range(3):
            for s in range(2):
                want = sorted(map(frozenset, mc_table.face_segments(c, a, s)), key=sorted)
                got = sorted(on_face.get((a, s), []), key=sorted)
                assert got == want, (c, a, s, got, want)


def test_ambiguous_face_rule_sees_only_the_face():
    """cubes sharing an ambiguous face pair its edges the same way: the rule depends on the face's four signs only"""
    for a in range(3):
        for c in range(256):
            segs = lambda cc, s: sorted(_face_key(seg, a) for seg in mc_table.face_segments(cc, a, s))
            # the neighbour along +a sees our side-1 face as its side-0 face: same corner signs, shifted by one along a
            nb = 0
            for b in range(8):
                if mc_table.CORNER[b][a] == 1 and c >> b & 1:
                    nb |= 1 << (b - (1 << a))
            assert segs(c, 1) == segs(nb, 0), (a, c)


def _face_key(seg, a):
    """a segment as the positions of its edge midpoints in the face plane (drops the coordinate along a)"""
    return tuple(sorted(tuple(np.delete(mc_table.EDGE_MID[e], a)) for e in seg))


# ------------------------------------------------------------------------------------------------ the whole-volume oracle
def _grid(n, lo=-1.0, hi=1.0):
    x = np.linspace(lo, hi, n)
    return np.stack(np.meshgrid(x, x, x, indexing="ij"), -1), (hi - lo) / (n - 1)


def _mc(sdf, h, lo=-1.0):
    return omesh.marching_cubes(sdf.astype(np.float32), 0.0, (lo, lo, lo), (h, h, h))


def _check_orientation(m, grad_fn):
    fn = omesh.face_normals(m["verts"], m["faces"])
    c = m["verts"][m["faces"]].mean(1)
    dots = (fn * grad_fn(c)).sum(1)
    assert (dots > 0).mean() > 0.999 and (dots * np.linalg.norm(fn, axis=1)).sum() > 0
    assert ((m["normals"] * grad_fn(m["verts"])).sum(1) > 0).all()


def test_sphere_closed_manifold_area_and_orientation():
    P, h = _grid(128)
    r = 0.7
    m = _mc(np.linalg.norm(P, axis=-1) - r, h)
    assert omesh.is_closed_oriented_manifold(m["faces"])
    assert omesh.euler_characteristic(m["verts"], m["faces"]) == 2
    assert abs(omesh.area(m["verts"], m["faces"]) / (4 * np.pi * r * r) - 1) < 0.01
    _check_orientation(m, lambda x: x)
    assert np.abs(np.linalg.norm(m["verts"], axis=1) - r).max() < h


def test_torus_euler_zero():
    P, h = _grid(96)
    R, r = 0.55, 0.2
    q = np.sqrt(P[..., 0] ** 2 + P[..., 1] ** 2) - R
    m = _mc(np.sqrt(q ** 2 + P[..., 2] ** 2) - r, h)
    assert omesh.is_closed_oriented_manifold(m["faces"])
    assert omesh.euler_characteristic(m["verts"], m["faces"]) == 0

    def grad(x):
        rho = np.sqrt(x[:, 0] ** 2 + x[:, 1] ** 2)
        return np.stack([x[:, 0] * (rho - R) / rho, x[:, 1] * (rho - R) / rho, x[:, 2]], 1)
    _check_orientation(m, grad)


def test_two_spheres_euler_four():
    P, h = _grid(80)
    c1, c2 = np.array([-0.45, 0, 0]), np.array([0.45, 0.1, 0])
    sdf = np.minimum(np.linalg.norm(P - c1, axis=-1), np.linalg.norm(P - c2, axis=-1)) - 0.3
    m = _mc(sdf, h)
    assert omesh.is_closed_oriented_manifold(m["faces"])
    assert omesh.euler_characteristic(m["verts"], m["faces"]) == 4

    def grad(x):
        d1, d2 = x - c1, x - c2
        return np.where((np.linalg.norm(d1, axis=1) < np.linalg.norm(d2, axis=1))[:, None], d1, d2)
    _check_orientation(m, grad)


def test_random_volume_is_a_closed_manifold_away_from_the_border():
    """every case and every ambiguous face occurs; edges inside the volume are shared by exactly two oppositely wound triangles"""
    rng = np.random.default_rng(0)
    vol = rng.standard_normal((12, 11, 13)).astype(np.float32)
    vol[0], vol[-1], vol[:, 0], vol[:, -1], vol[:, :, 0], vol[:, :, -1] = 1, 1, 1, 1, 1, 1      # outside on the border: a closed mesh
    m = omesh.marching_cubes(vol, 0.0)
    assert len(np.unique(m["cases"])) > 200
    assert omesh.is_closed_oriented_manifold(m["faces"])


def test_oracle_vertex_order_and_formula():
    rng = np.random.default_rng(1)
    vol = rng.standard_normal((5, 4, 6)).astype(np.float32)
    m = omesh.marching_cubes(vol, 0.25, (1.0, -2.0, 0.5), (0.5, 0.25, 2.0))
    e = m["edge"]
    assert (np.lexsort(e.T[::-1]) == np.arange(len(e))).all()                 # (i, j, k, axis) order
    i, j, k, a = e[0]
    q = e[0, :3] + np.eye(3, dtype=int)[a]
    t = (0.25 - float(vol[i, j, k])) / (float(vol[tuple(q)]) - float(vol[i, j, k]))
    want = np.array([1.0, -2.0, 0.5]) + np.array([0.5, 0.25, 2.0]) * (e[0, :3] + t * np.eye(3)[a])
    assert np.array_equal(m["verts"][0], want)


# ------------------------------------------------------------------------------------------------ PLY writer
def _parse_ply(path):
    with open(path, "rb") as f:
        data = f.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    return data[:end].decode("ascii"), data[end:]


@pytest.mark.parametrize("with_color", [False, True])
def test_ply_round_trip(tmp_path, with_color):
    from neuralsim_b200.graphics.trianglemesh import write_ply
    rng = np.random.default_rng(2)
    V, F = 7, 5
    verts = rng.standard_normal((V, 3)).astype(np.float32)
    faces = rng.integers(0, V, (F, 3)).astype(np.int32)
    colors = rng.integers(0, 256, (V, 3)).astype(np.uint8) if with_color else None
    p = str(tmp_path / "m.ply")
    write_ply(p, verts, faces, colors)
    header, body = _parse_ply(p)
    want = ("ply\nformat binary_little_endian 1.0\nelement vertex 7\nproperty float x\nproperty float y\nproperty float z\n"
            + ("property uchar red\nproperty uchar green\nproperty uchar blue\n" if with_color else "")
            + "element face 5\nproperty list uchar int vertex_indices\nend_header\n")
    assert header == want
    vdt = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")] + ([("red", "u1"), ("green", "u1"), ("blue", "u1")] if with_color else [])
    nvb = np.dtype(vdt).itemsize * V
    v = np.frombuffer(body[:nvb], dtype=vdt)
    f = np.frombuffer(body[nvb:], dtype=[("n", "u1"), ("vertex_indices", "<i4", (3,))])
    assert len(body) == nvb + 13 * F
    assert np.array_equal(np.stack([v["x"], v["y"], v["z"]], 1), verts)
    assert (f["n"] == 3).all() and np.array_equal(f["vertex_indices"], faces)
    if with_color:
        assert np.array_equal(np.stack([v["red"], v["green"], v["blue"]], 1), colors)
