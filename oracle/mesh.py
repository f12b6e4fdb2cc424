"""float64 numpy restatement of the marching-cubes stages of csrc/mesh.cu on a whole volume (no slabs), with the same case table
(oracle/mc_table.py) and the same vertex and triangle order:
  vertices  one per lattice edge whose ends differ in sign (inside: sdf < level), in (i, j, k, axis) order of the edge's owner point;
            position bmin + spacing (idx + t), t = (level - s0) / (s1 - s0); normal = normalise(g0 + t (g1 - g0)) of the lattice gradient
            (central differences, one-sided at the volume border, over the spacing);
  faces     the case table's triangles of every cell in (i, j, k) order, as vertex ids.
"""
from __future__ import annotations

import numpy as np

from . import mc_table


def lattice_gradient(vol, spacing):
    """[n0, n1, n2, 3]: d vol / d axis, central differences inside, one-sided at the border, over the spacing"""
    vol = np.asarray(vol, dtype=np.float64)
    g = np.empty(vol.shape + (3,))
    for a in range(3):
        v = np.moveaxis(vol, a, 0)
        d = np.empty_like(v)
        d[1:-1] = (v[2:] - v[:-2]) / (2.0 * spacing[a])
        d[0] = (v[1] - v[0]) / spacing[a]
        d[-1] = (v[-1] - v[-2]) / spacing[a]
        g[..., a] = np.moveaxis(d, 0, a)
    return g


def marching_cubes(vol, level=0.0, bmin=(0., 0., 0.), spacing=(1., 1., 1.)):
    """-> dict(verts [V,3] f64, normals [V,3] f64, faces [F,3] int64, edge [V,4] int64 = (i, j, k, axis) of each vertex's lattice edge,
    cases [n0-1, n1-1, n2-1] uint8)"""
    vol = np.asarray(vol, dtype=np.float64)
    n0, n1, n2 = vol.shape
    assert min(vol.shape) >= 2
    bmin, spacing = np.asarray(bmin, np.float64), np.asarray(spacing, np.float64)
    inside = vol < level
    flags = np.zeros(vol.shape + (3,), dtype=bool)
    flags[:-1, :, :, 0] = inside[:-1] != inside[1:]
    flags[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    flags[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    vid = np.cumsum(flags.reshape(-1)).reshape(flags.shape) - 1          # vertex id of each set (point, axis)
    edge = np.argwhere(flags)                                             # C order = (i, j, k, axis) order
    p, a = edge[:, :3], edge[:, 3]
    q = p + np.eye(3, dtype=np.int64)[a]
    s0, s1 = vol[p[:, 0], p[:, 1], p[:, 2]], vol[q[:, 0], q[:, 1], q[:, 2]]
    t = (level - s0) / (s1 - s0)
    idx = p.astype(np.float64)
    idx[np.arange(len(a)), a] += t
    verts = bmin + spacing * idx
    G = lattice_gradient(vol, spacing)
    g0, g1 = G[p[:, 0], p[:, 1], p[:, 2]], G[q[:, 0], q[:, 1], q[:, 2]]
    nrm = g0 + t[:, None] * (g1 - g0)
    nn = np.sqrt((nrm * nrm).sum(1, keepdims=True))
    normals = np.where(nn > 0, nrm / np.where(nn > 0, nn, 1.0), 0.0)

    count, table = mc_table.build_table()
    case = np.zeros((n0 - 1, n1 - 1, n2 - 1), dtype=np.int64)
    for b in range(8):
        dx, dy, dz = mc_table.CORNER[b]
        case |= inside[dx:dx + n0 - 1, dy:dy + n1 - 1, dz:dz + n2 - 1].astype(np.int64) << b
    cnt = count[case.reshape(-1)]
    cells = np.repeat(np.arange(case.size), cnt)
    entry = np.arange(cells.size) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    ci = np.stack(np.unravel_index(cells, case.shape), 1)
    e = table[case.reshape(-1)[cells][:, None], 3 * entry[:, None] + np.arange(3)[None, :]]       # [F, 3] edge ids
    owner = ci[:, None, :] + np.asarray(mc_table.EDGE_OWNER, dtype=np.int64)[e]
    axis = np.asarray(mc_table.EDGE_AXIS, dtype=np.int64)[e]
    faces = vid[owner[..., 0], owner[..., 1], owner[..., 2], axis]
    return dict(verts=verts, normals=normals, faces=faces.reshape(-1, 3), edge=edge, cases=case.astype(np.uint8))


def mesh_edges(faces):
    """directed edges (a, b) of every triangle, [3F, 2]"""
    f = np.asarray(faces)
    return np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])


def euler_characteristic(verts, faces):
    f = np.asarray(faces)
    und = np.sort(mesh_edges(f), 1)
    n_edges = np.unique(und, axis=0).shape[0]
    n_verts = np.unique(f).size
    return n_verts - n_edges + f.shape[0]


def is_closed_oriented_manifold(faces):
    """every undirected edge in exactly two triangles, traversed in opposite directions"""
    d = mesh_edges(faces)
    und = np.sort(d, 1)
    _, inv, cnt = np.unique(und, axis=0, return_inverse=True, return_counts=True)
    if not np.all(cnt == 2):
        return False
    _, dcnt = np.unique(d, axis=0, return_counts=True)
    return bool(np.all(dcnt == 1))


def face_normals(verts, faces):
    v = np.asarray(verts)[np.asarray(faces)]
    return np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0])


def area(verts, faces):
    return float(0.5 * np.linalg.norm(face_normals(verts, faces), axis=1).sum())
