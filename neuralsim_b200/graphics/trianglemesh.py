"""Mesh extraction on the GPU: `nr3d_lib.graphics.trianglemesh.extract_mesh` (trianglemesh.py:134-254) with the lattice streamed through
the SDF query in slabs of whole planes and marching cubes in CUDA (csrc/mesh.cu), plus a vectorised binary PLY writer.

The reference builds the whole lattice on the host, copies every 16 Ki-point chunk of SDF values back into a float64 numpy volume, runs
skimage's marching cubes on the CPU and writes the PLY file one Python iteration per element.  Here the lattice points of a slab are made on
the device, queried in calls of at most `chunk` points, and the slab's vertices and triangles are emitted before the next slab is queried;
the host reads two totals per slab (to size the outputs).  The output order is fixed by exclusive scans -- vertices in (i, j, k, axis) order
of the lattice edge they lie on, triangles in (cell, table entry) order -- so the result does not depend on `chunk` and two runs agree bit
for bit.  Vertex positions follow skimage's interpolation (`spacing = (bmax - bmin) / (N - 1)`, position `bmin + spacing (idx + t)`); in a
cell with an ambiguous face the triangulation is this package's (the face's inside corners are separated: oracle/mc_table.py), not
skimage's Lewiner tables.
"""
from __future__ import annotations

import ctypes
import sys
import time
from typing import Callable, List, Union

import numpy as np
import torch

from .. import _lib as L
from .neus_fused import _scan_ws_bytes, scan_counts, scan_launch

__all__ = ["extract_mesh", "write_ply"]

MC_MAX_TRIS = 5                                  # kMcMaxTris of csrc/mc_table.cuh: triangles of one cell at most
_I32_MAX = 2 ** 31 - 1
_SLAB_MAX_SLOTS = _I32_MAX // MC_MAX_TRIS        # a slab's scanned offsets are int32


def _ply_header(n_verts, n_faces, with_color):
    props = ["x", "y", "z"]
    lines = ["ply", "format binary_little_endian 1.0", f"element vertex {n_verts}"] + [f"property float {p}" for p in props]
    if with_color:
        lines += [f"property uchar {p}" for p in ("red", "green", "blue")]
    lines += [f"element face {n_faces}", "property list uchar int vertex_indices", "end_header"]
    return ("\n".join(lines) + "\n").encode("ascii")


def write_ply(filepath, verts, faces, colors=None):
    """Binary little-endian PLY with the element and property names the reference writes through plyfile: vertex x y z (float) [+ red green
    blue (uchar)], face `vertex_indices` (list uchar int).  verts [V, 3] float32, faces [F, 3] int32, colors [V, 3] uint8 or None (numpy or
    tensors).  The body is built from numpy structured arrays and written with one call."""
    as_np = lambda a: a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    verts, faces = as_np(verts).reshape(-1, 3), as_np(faces).reshape(-1, 3)
    vdt = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    if colors is not None:
        vdt += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    v = np.empty(verts.shape[0], dtype=vdt)
    for q, name in enumerate("xyz"):
        v[name] = verts[:, q]
    if colors is not None:
        colors = as_np(colors).reshape(-1, 3)
        for q, name in enumerate(("red", "green", "blue")):
            v[name] = colors[:, q]
    f = np.empty(faces.shape[0], dtype=[("n", "u1"), ("vertex_indices", "<i4", (3,))])
    f["n"] = 3
    f["vertex_indices"] = faces
    with open(filepath, "wb") as fh:
        fh.write(b"".join((_ply_header(v.shape[0], f.shape[0], colors is not None), v.tobytes(), f.tobytes())))


def _lattice_dims(bmin, bmax, N):
    volume_size = bmax - bmin
    if isinstance(N, (int, np.integer)) or len(N) == 1:
        N = (volume_size / volume_size.min() * N).astype(np.int32)
    else:
        N = np.array(N)
    return N


@torch.no_grad()
def extract_mesh(
        query_sdf_fn: Callable[[torch.Tensor], torch.Tensor],
        query_color_fn: Callable[[torch.Tensor, torch.Tensor], torch.Tensor] = None, *,
        filepath: str = "./surface.ply",
        level: float = 0.0, N: Union[int, List[int]] = 512, chunk: int = 16 * 1024,
        include_color=False, show_progress=True,
        bmin: Union[List, np.ndarray] = [-1., -1., -1.], bmax: Union[List, np.ndarray] = [1., 1., 1.],
        offset: np.ndarray = None, scale: np.ndarray = None, transform: np.ndarray = None,
        device=torch.device("cuda")):
    """Marching cubes of the level set `query_sdf_fn(x) == level` on an N-point lattice of [bmin, bmax]; writes a PLY file.

    Same arguments as the reference's extract_mesh:
      N: lattice points per axis, or an int: the count along the shortest side of the box, `(size / size.min() * N).astype(int32)`.
         The axis vectors are CPU float32 `torch.linspace(bmin[a], bmax[a], N[a])`, so every queried point equals the reference's `xyz`
         row bit for bit.
      chunk: the most points one `query_sdf_fn` (and `query_color_fn`) call receives.  A slab holds max(1, chunk // (N[1] N[2])) planes.
      query_color_fn(x, v): called on the vertices in device chunks with v = -normal, the unit direction of a ray that reaches the surface
         from outside (sdf >= level) -- the view direction the radiance net was trained on.  (The reference passes skimage's normals; their
         sign convention is not checked against this choice.)  colours = (rgb * 255).to(uint8).
      scale, offset, transform: applied after the colour query, in float64, in this order: `v * scale`, `v - offset`,
         `v @ transform[:3, :3].T + transform[:3, 3]`; then cast to float32.
      filepath: None skips the file.
    A point is inside when sdf < level.  SDF values are held as float32 (fp16 and fp32 queries lose nothing).  Face winding: the right-hand
    normal points along +grad sdf.  Vertex normals: central differences of the lattice SDF (one-sided at the volume border) over the
    spacing, interpolated along the edge and normalised (unchanged by scale / offset / transform).

    -> dict(verts [V, 3] float32, faces [F, 3] int32, normals [V, 3] float32, colors [V, 3] uint8 or None, timing: seconds per stage
       {query, marching_cubes, color, ply}), all tensors on `device`."""
    t_start = time.perf_counter()
    dev = torch.device(device)
    bmin, bmax = np.array(bmin, dtype=np.float64), np.array(bmax, dtype=np.float64)
    N = _lattice_dims(bmin, bmax, N)
    n0, n1, n2 = (int(v) for v in N)
    if min(n0, n1, n2) < 2:
        raise ValueError(f"extract_mesh: the lattice needs >= 2 points per axis, got {n0} x {n1} x {n2}")
    spacing = (bmax - bmin) / (N - 1)
    plane = n1 * n2
    if plane > _SLAB_MAX_SLOTS:
        raise ValueError(f"extract_mesh: a lattice plane of {n1} x {n2} points is too large for int32 offsets")
    chunk = int(chunk)
    if chunk < 1:
        raise ValueError("extract_mesh: chunk must be >= 1")
    lin = [torch.linspace(bmin[a], bmax[a], int(N[a])).to(dev) for a in range(3)]
    S = max(1, min(chunk // plane, _SLAB_MAX_SLOTS // plane, n0))
    lib, stream = L.lib(), L.stream_ptr()
    bmin_c, spacing_c = (ctypes.c_double * 3)(*bmin.tolist()), (ctypes.c_double * 3)(*spacing.tolist())

    win = torch.empty((S + 3) * plane, dtype=torch.float32, device=dev)     # sdf of planes [h0, h1): a slab and its halo
    x = torch.empty(min(chunk, n0 * plane), 3, dtype=torch.float32, device=dev)
    flags_b = torch.empty(S * plane, dtype=torch.uint8, device=dev)
    cases_b = torch.empty(S * plane, dtype=torch.uint8, device=dev)
    vcount_b = torch.empty(S * plane, dtype=torch.int32, device=dev)
    tcount_b = torch.empty(S * plane, dtype=torch.int32, device=dev)
    vfirst_b = torch.empty(S * plane, dtype=torch.int32, device=dev)
    vtot = torch.zeros(4, dtype=torch.int64, device=dev)
    ws_bytes = _scan_ws_bytes()
    carry_flags = carry_first = None
    carry_base = vbase = 0
    h0 = h1 = 0
    verts_l, normals_l, faces_l = [], [], []
    ev = []                                                  # (start, after query, after marching cubes) per slab
    n_slabs = (n0 + S - 1) // S
    for si, p0 in enumerate(range(0, n0, S)):
        p1 = min(p0 + S, n0)
        w0, w1 = max(p0 - 1, 0), min(p1 + 2, n0)             # one plane before the slab (its cells), two after (the last +x edges' normals)
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e[0].record()
        start = w0
        if h1 > w0:                                          # the planes already queried for the previous slab move to the front
            keep = win[(w0 - h0) * plane:(h1 - h0) * plane].clone()
            win[:keep.numel()].copy_(keep)
            start = h1
        h0, h1 = w0, w1
        for s in range(start * plane, w1 * plane, chunk):
            m = min(s + chunk, w1 * plane) - s
            L.check(lib.nsb_mc_lattice_points(L.ptr(lin[0]), L.ptr(lin[1]), L.ptr(lin[2]), n1, n2, s, m, L.ptr(x), stream), "mc_lattice_points")
            sdf = query_sdf_fn(x[:m])
            if sdf.numel() != m:
                raise RuntimeError(f"extract_mesh: query_sdf_fn returned {sdf.numel()} values for {m} points")
            win[s - w0 * plane:s - w0 * plane + m].copy_(sdf.reshape(-1))
        e[1].record()

        n = (p1 - p0) * plane
        flags, cases, vcount, tcount, vfirst = flags_b[:n], cases_b[:n], vcount_b[:n], tcount_b[:n], vfirst_b[:n]
        L.check(lib.nsb_mc_count(L.ptr(win), w0, w1 - w0, n0, n1, n2, p0, p1, float(level), L.ptr(flags), L.ptr(vcount), L.ptr(cases),
                                 L.ptr(tcount), stream), "mc_count")
        ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=dev)
        scan_launch(vcount, L.ptr(vtot), first=vfirst, ws=ws)
        sc = scan_counts(tcount, want_first=True, extra=vtot[:1])        # the slab's one host read: triangle and vertex totals
        nt, nv = sc["total"], sc["extra"][0]
        if vbase + nv > _I32_MAX:
            raise RuntimeError(f"extract_mesh: more than 2^31 - 1 vertices ({vbase + nv} by plane {p1}): int32 face indices would overflow")
        verts = torch.empty(nv, 3, dtype=torch.float32, device=dev)
        normals = torch.empty(nv, 3, dtype=torch.float32, device=dev)
        faces = torch.empty(nt, 3, dtype=torch.int32, device=dev)
        if nv:
            L.check(lib.nsb_mc_vertices(L.ptr(win), w0, w1 - w0, n0, n1, n2, p0, p1, float(level), bmin_c, spacing_c, L.ptr(flags),
                                        L.ptr(vfirst), L.ptr(verts), L.ptr(normals), stream), "mc_vertices")
        if nt:
            L.check(lib.nsb_mc_triangles(n0, n1, n2, p0, p1, L.ptr(cases), L.ptr(tcount), L.ptr(sc["first"]), L.ptr(flags), L.ptr(vfirst), vbase,
                                         L.ptr(carry_flags, allow_none=True), L.ptr(carry_first, allow_none=True), carry_base, L.ptr(faces),
                                         stream), "mc_triangles")
        carry_flags, carry_first, carry_base = flags[n - plane:].clone(), vfirst[n - plane:].clone(), vbase
        vbase += nv
        verts_l.append(verts)
        normals_l.append(normals)
        faces_l.append(faces)
        e[2].record()
        ev.append(e)
        if show_progress:
            print(f"\rextract_mesh: slab {si + 1}/{n_slabs}, {vbase} vertices", end="", file=sys.stderr, flush=True)
    if show_progress:
        print(file=sys.stderr)
    verts, normals, faces = torch.cat(verts_l), torch.cat(normals_l), torch.cat(faces_l)
    torch.cuda.synchronize(dev)
    timing = dict(query=sum(a.elapsed_time(b) for a, b, _ in ev) / 1e3, marching_cubes=sum(b.elapsed_time(c) for _, b, c in ev) / 1e3)

    t0 = time.perf_counter()
    colors = None
    if include_color:
        if query_color_fn is None:
            raise ValueError("extract_mesh: include_color needs query_color_fn")
        colors = torch.empty(verts.shape[0], 3, dtype=torch.uint8, device=dev)
        for s in range(0, verts.shape[0], chunk):
            rgb = query_color_fn(verts[s:s + chunk], -normals[s:s + chunk])
            colors[s:s + chunk] = (rgb * 255.).to(torch.uint8)
    if scale is not None or offset is not None or transform is not None:
        v64 = verts.double()
        if scale is not None:
            v64 = v64 * torch.from_numpy(np.array(scale, dtype=np.float32)).to(dev).double()
        if offset is not None:
            v64 = v64 - torch.from_numpy(np.array(offset, dtype=np.float32)).to(dev).double()
        if transform is not None:
            T = torch.from_numpy(np.array(transform, dtype=np.float32)).to(dev).double()
            v64 = v64 @ T[:3, :3].T + T[:3, 3]
        verts = v64.float()
    torch.cuda.synchronize(dev)
    timing["color"] = time.perf_counter() - t0

    t0 = time.perf_counter()
    if filepath is not None:
        write_ply(filepath, verts, faces, colors)
    timing["ply"] = time.perf_counter() - t0
    timing["total"] = time.perf_counter() - t_start
    return dict(verts=verts, faces=faces, normals=normals, colors=colors, timing=timing)
