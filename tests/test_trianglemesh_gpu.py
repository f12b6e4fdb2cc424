"""GPU marching cubes (csrc/mesh.cu behind neuralsim_b200.graphics.trianglemesh.extract_mesh) against the float64 whole-volume oracle
(oracle/mesh.py) on stored volumes, slab invariance, and meshes of the CFG sphere model and the cfg3 road plane.

A stored volume is queried on the lattice bmin = 0, bmax = N - 1: the lattice coordinates are exact integers and index the volume."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import mesh as omesh

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _volume_query(vol, device):
    V = torch.from_numpy(np.ascontiguousarray(vol, dtype=np.float32)).to(device)

    def q(x):
        i = x.long()
        assert torch.equal(i.float(), x)
        return V[i[:, 0], i[:, 1], i[:, 2]]
    return q


def _extract(vol, device, level=0.0, chunk=None, **kw):
    from neuralsim_b200.graphics.trianglemesh import extract_mesh
    n = list(vol.shape)
    return extract_mesh(_volume_query(vol, device), filepath=None, level=level, N=n, chunk=chunk or int(np.prod(n)), show_progress=False,
                        bmin=[0., 0., 0.], bmax=[float(v - 1) for v in n], device=device, **kw)


def _assert_matches_oracle(out, vol, level=0.0, bmin=(0., 0., 0.), spacing=(1., 1., 1.)):
    ref = omesh.marching_cubes(vol, level, bmin, spacing)
    faces = out["faces"].cpu().numpy()
    verts, normals = out["verts"].cpu().numpy(), out["normals"].cpu().numpy()
    assert faces.dtype == np.int32 and verts.dtype == np.float32
    assert verts.shape == ref["verts"].shape and faces.shape == ref["faces"].shape
    assert np.array_equal(faces.astype(np.int64), ref["faces"])
    # vertex q of both lies on lattice edge ref["edge"][q]: the same order; positions within 2 fp32 ulps of the float64 value
    ulp = np.spacing(np.abs(ref["verts"]).astype(np.float32)).astype(np.float64)
    err = np.abs(verts.astype(np.float64) - ref["verts"])
    assert (err <= 2 * ulp).all(), (err / ulp).max()
    assert np.abs(normals.astype(np.float64) - ref["normals"]).max(initial=0.0) <= 1e-5
    return ref


def _grid(shape, c=None):
    ax = [np.arange(n, dtype=np.float64) for n in shape]
    P = np.stack(np.meshgrid(*ax, indexing="ij"), -1)
    return P - (np.array(shape, dtype=np.float64) - 1) / 2 if c is None else P - np.asarray(c, dtype=np.float64)


def _sphere(shape, r, c=None):
    return (np.linalg.norm(_grid(shape, c), axis=-1) - r).astype(np.float32)


def _torus(shape, R, r):
    P = _grid(shape)
    q = np.sqrt(P[..., 0] ** 2 + P[..., 1] ** 2) - R
    return (np.sqrt(q ** 2 + P[..., 2] ** 2) - r).astype(np.float32)


VOLUMES = {
    "sphere_odd": lambda: _sphere((33, 40, 29), 11.3),
    "torus": lambda: _torus((48, 44, 20), 13.0, 5.2),
    "random": lambda: np.random.default_rng(0).standard_normal((17, 19, 23)).astype(np.float32),
    "exact_level_ints": lambda: np.random.default_rng(1).integers(-1, 2, (13, 9, 11)).astype(np.float32),
    "exact_level_sphere": lambda: np.round(_sphere((21, 22, 23), 7.0) * 2) / 2,
    "cut_by_box": lambda: _sphere((24, 30, 18), 14.0, c=(3.0, 25.0, 9.0)),
    "plane_open": lambda: (_grid((12, 15, 10))[..., 2] - 0.37).astype(np.float32),
    "cube_2x2x2": lambda: np.random.default_rng(2).standard_normal((2, 2, 2)).astype(np.float32),
    "thin_2x7x3": lambda: np.random.default_rng(3).standard_normal((2, 7, 3)).astype(np.float32),
    "thin_5x2x9": lambda: np.random.default_rng(4).standard_normal((5, 2, 9)).astype(np.float32),
}


@pytest.mark.parametrize("name", sorted(VOLUMES))
def test_volume_matches_oracle(cuda, name):
    vol = VOLUMES[name]()
    out = _extract(vol, cuda)
    ref = _assert_matches_oracle(out, vol)
    if name in ("sphere_odd", "torus"):
        assert omesh.is_closed_oriented_manifold(ref["faces"])
        assert omesh.euler_characteristic(ref["verts"], ref["faces"]) == (2 if name == "sphere_odd" else 0)
    if name == "cut_by_box":
        assert not omesh.is_closed_oriented_manifold(ref["faces"]) and ref["faces"].shape[0] > 0


def test_random_volume_at_a_level(cuda):
    vol = np.random.default_rng(5).standard_normal((16, 12, 14)).astype(np.float32)
    _assert_matches_oracle(_extract(vol, cuda, level=0.3), vol, level=0.3)


def test_all_2x2x2_cases(cuda):
    """the 256 corner-sign cases of one cell, each as its own 2 x 2 x 2 volume (values -1 / +1 and exact zeros)"""
    for c in range(256):
        vol = np.array([-1.0 if c >> b & 1 else (0.0 if b % 3 == 0 else 1.0) for b in range(8)], dtype=np.float32)
        vol = vol.reshape(2, 2, 2).transpose(2, 1, 0).copy()            # corner b at (b & 1, b >> 1 & 1, b >> 2 & 1)
        _assert_matches_oracle(_extract(vol, cuda), vol)


@pytest.mark.parametrize("fill", [-1.0, 1.0])
def test_all_inside_or_outside_is_empty(cuda, fill):
    vol = np.full((9, 6, 7), fill, dtype=np.float32)
    out = _extract(vol, cuda)
    assert out["verts"].shape == (0, 3) and out["faces"].shape == (0, 3) and out["normals"].shape == (0, 3)


@pytest.mark.parametrize("name", ["torus", "random", "cut_by_box"])
def test_slab_size_changes_nothing(cuda, name):
    vol = VOLUMES[name]()
    n0, n1, n2 = vol.shape
    plane = n1 * n2
    runs = [_extract(vol, cuda, chunk=c) for c in (n2, plane, 2 * plane + n2, 3 * plane, n0 * plane, n0 * plane)]
    for r in runs[1:]:
        for k in ("verts", "normals", "faces"):
            assert torch.equal(r[k], runs[0][k]), k


def test_include_color(cuda):
    vol = VOLUMES["sphere_odd"]()
    color_fn = lambda x, v: torch.sigmoid(0.1 * x + v[:, [2, 0, 1]])
    out = _extract(vol, cuda, chunk=1000, include_color=True, query_color_fn=color_fn)
    want = (color_fn(out["verts"], -out["normals"]) * 255.).to(torch.uint8)
    assert out["colors"].dtype == torch.uint8 and torch.equal(out["colors"], want)


def test_transform_and_ply_file(cuda, tmp_path):
    vol = VOLUMES["torus"]()
    base = _extract(vol, cuda)
    scale, offset = np.array([2.0, 0.5, 1.5]), np.array([1.0, -2.0, 0.25])
    T = np.eye(4)
    T[:3, :3] = [[0, -1, 0], [1, 0, 0], [0, 0, 1]]
    T[:3, 3] = [3.0, 4.0, 5.0]
    p = str(tmp_path / "t.ply")
    from neuralsim_b200.graphics.trianglemesh import extract_mesh
    n = list(vol.shape)
    out = extract_mesh(_volume_query(vol, cuda), filepath=p, N=n, show_progress=False, bmin=[0., 0., 0.], bmax=[float(v - 1) for v in n],
                       scale=scale, offset=offset, transform=T, device=cuda)
    v64 = base["verts"].cpu().double().numpy() * scale.astype(np.float32) - offset.astype(np.float32)
    v64 = v64 @ T.astype(np.float32)[:3, :3].T.astype(np.float64) + T.astype(np.float32)[:3, 3]
    assert np.array_equal(out["verts"].cpu().numpy(), v64.astype(np.float32))
    with open(p, "rb") as f:
        data = f.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    V, F = out["verts"].shape[0], out["faces"].shape[0]
    assert f"element vertex {V}\n".encode() in data[:end] and f"element face {F}\n".encode() in data[:end]
    assert np.array_equal(np.frombuffer(data[end:end + 12 * V], "<f4").reshape(V, 3), out["verts"].cpu().numpy())


def test_vertex_count_overflow_raises_before_emitting(cuda, monkeypatch):
    from neuralsim_b200.graphics import trianglemesh as TM
    vol = VOLUMES["random"]()
    monkeypatch.setattr(TM, "_I32_MAX", 100)
    with pytest.raises(RuntimeError, match="int32"):
        _extract(vol, cuda)


# ------------------------------------------------------------------------------------------------ models
def _lattice_volume(q, bmin, bmax, N, device):
    lin = [torch.linspace(bmin[a], bmax[a], N[a]).to(device) for a in range(3)]
    xyz = torch.stack(torch.meshgrid(*lin, indexing="ij"), -1).reshape(-1, 3)
    with torch.no_grad():
        return torch.cat([q(xyz[s:s + 65536]).reshape(-1).float() for s in range(0, xyz.shape[0], 65536)]).view(*N).cpu().numpy()


def test_cfg_sphere_model_matches_oracle_on_its_volume(cuda):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from util import make_pair
    from neuralsim_b200.graphics.trianglemesh import extract_mesh
    _, model = make_pair(cuda)
    model.eval()
    assert model.implicit_surface._fusable()
    q = lambda x: model.forward_sdf(model.space.normalize_coords(x))["sdf"]
    N = [40, 44, 36]
    bmin, bmax = np.array([-1., -1., -1.]), np.array([1., 1., 1.])
    out = extract_mesh(q, filepath=None, N=N, chunk=5000, bmin=bmin, bmax=bmax, show_progress=False, device=cuda)
    vol = _lattice_volume(q, bmin, bmax, N, cuda)
    ref = _assert_matches_oracle(out, vol, 0.0, bmin, (bmax - bmin) / (np.array(N) - 1))
    assert ref["faces"].shape[0] > 1000
    r = np.linalg.norm(ref["verts"], axis=1)
    assert np.abs(r - 0.5).max() < 0.05


@pytest.mark.parametrize("levels", [16, 17])
def test_cfg3_road_plane(cuda, levels):
    sys.path.insert(0, ROOT)
    import bench_cfg3 as C
    from neuralsim_b200.graphics.trianglemesh import extract_mesh
    model = C.build_model(cuda, max_num_levels=levels, log2_hashmap_size=16, target_num_params=(levels + 2) * 2 ** 17).eval()
    assert model.implicit_surface._fusable() == (levels == 16)
    q = lambda x: model.forward_sdf(model.space.normalize_coords(x))["sdf"]
    bmin, bmax = [-6., -12., -7.5], [6., 12., -3.5]
    out = extract_mesh(q, filepath=None, N=24, chunk=20000, bmin=bmin, bmax=bmax, show_progress=False, device=cuda)
    v, nrm = out["verts"].cpu().numpy(), out["normals"].cpu().numpy()
    assert v.shape[0] > 1000
    dz = np.abs(v[:, 2] - C.ROAD_Z)
    print(f"levels {levels}: {v.shape[0]} vertices, max |z - ROAD_Z| {dz.max():.2e} m, min normal z {nrm[:, 2].min():.4f}")
    assert dz.max() < 0.02          # the table's random detail reaches the decoded sdf: ~1 cm off the installed plane on this seed
    assert nrm[:, 2].min() > 0.99
    f = out["faces"].cpu().numpy().astype(np.int64)
    assert (omesh.face_normals(v, f)[:, 2] > 0).all()
