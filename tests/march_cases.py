"""Inputs of the marcher's edge tests (tests/test_march_edges_gpu.py, tests/test_march_oracle.py), generated on the CPU from fixed seeds.

The street geometry is cfg3's (bench_cfg3.py): the 40 x 150 x 15 m cuboid, rays in metres normalised by its per-axis half size as the
NeuS step normalises them (fields/space.py: normalize_rays), step 0.2 m, max_steps 4096, near / far from the ray test (oracle/render.py).
Every ray has a direction with a non-zero component and a finite far, so the marcher's voxel-skipping loop always ends."""
import math

import numpy as np
import torch

from oracle import render as orender

HALF = np.array([20.0, 75.0, 7.5])          # metres; the box is centred on the origin
EGO_Z = -3.5                                # 2 m above cfg3's road (ROAD_Z = -5.5)
NEAR, FAR = 0.1, 200.0
STEP, MAX_STEPS = 0.2, 4096
SMALL, LARGE = (40, 150, 15), (100, 375, 37)      # 1 m voxels (90 000 cells: not a multiple of 32, shared memory); 0.4 m (global memory)
SMEM_EDGE, GLOBAL_EDGE = (64, 96, 128), (65, 96, 128)   # exactly 786 432 cells (96 KB of bits, the last shared-memory size); one plane more
ROI = (-1., -1., -1., 1., 1., 1.)
ROI_FACE = (-1., -1., -1., 0.5, 1., 1.)    # a sub-box whose x-max face the roi-face rays lie on (world x = 10 m)


def _unit(d):
    return d / np.linalg.norm(d, axis=-1, keepdims=True)


def camera(H, W, pos, fwd_sign, focal):
    """a pinhole camera at pos looking along fwd_sign * y with the image rows along -z.  Pixels are offset from the centre without the
    half-pixel shift, so the centre row has dz = -0.0 and the centre column dx = +-0.0 exactly"""
    j, i = np.meshgrid(np.arange(H) - H // 2, np.arange(W) - W // 2, indexing="ij")
    x, z = (i / focal) * fwd_sign, -(j / focal)
    d = _unit(np.stack([x, np.full(x.shape, float(fwd_sign)), z], -1).reshape(-1, 3))
    return np.broadcast_to(np.asarray(pos, np.float64), d.shape), d


def lidar(pos, n_azim):
    """a 64-beam fan: 62 elevations from -17.6 to +2.4 deg and two horizontal beams with dz = +0.0 and dz = -0.0 exactly"""
    elev = np.concatenate([np.radians(np.linspace(-17.6, 2.4, 62)), [0.0, -0.0]])
    azim = 2 * math.pi * np.arange(n_azim) / n_azim
    e, a = np.meshgrid(elev, azim, indexing="ij")
    d = np.stack([np.cos(e) * np.sin(a), np.cos(e) * np.cos(a), np.sin(e)], -1).reshape(-1, 3)
    return np.broadcast_to(np.asarray(pos, np.float64), d.shape), d


def axis_rays(rng, n):
    """n origins inside the box, each with the six axis directions"""
    o = rng.uniform(-0.9, 0.9, (n, 3)) * HALF
    dirs = np.concatenate([np.eye(3), -np.eye(3)])
    return np.repeat(o, 6, 0), np.tile(dirs, (n, 1))


def boundary_rays(rng, n):
    """origins on a face (x = +20 m), an edge (x = +20, y = -75) and a corner (+20, -75, -7.5), with inward directions"""
    os_, ds_ = [], []
    for fixed in ((0,), (0, 1), (0, 1, 2)):
        o = rng.uniform(-0.9, 0.9, (n, 3)) * HALF
        d = _unit(rng.normal(size=(n, 3)))
        for k in fixed:
            s = 1.0 if k == 0 else -1.0
            o[:, k] = s * HALF[k]
            d[:, k] = -s * np.maximum(np.abs(d[:, k]), 0.05)
        os_.append(o); ds_.append(_unit(d))
    return np.concatenate(os_), np.concatenate(ds_)


def roi_face_rays(rng, n):
    """axis-parallel rays (+-y, +-z) lying on the x-max face of ROI_FACE"""
    o = rng.uniform(-0.9, 0.9, (n, 3)) * HALF
    o[:, 0] = 0.5 * HALF[0]
    dirs = np.array([[0., 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]])
    return np.repeat(o, 4, 0), np.tile(dirs, (n, 1))


def tested(o, d):
    """world rays (metres) -> normalised float32 rays and near / far of the ray test, as the NeuS step (rays that miss the box dropped)"""
    h = torch.tensor(HALF, dtype=torch.float32)
    o = (torch.from_numpy(np.ascontiguousarray(o, np.float32))) / h
    d = torch.from_numpy(np.ascontiguousarray(d, np.float32)) / h
    rt = orender.ray_test(o, d, near=NEAR, far=FAR)
    return tuple(rt[k].contiguous() for k in ("rays_o", "rays_d", "near", "far"))


def street_rays(n_azim=2000, cam_hw=(48, 64), n_axis=64, n_boundary=128, seed=0):
    """ego cameras inside the box along +-y, a LiDAR fan, axis-parallel rays, rays from a face / edge / corner, rays on ROI_FACE's face"""
    rng = np.random.default_rng(seed)
    H, W = cam_hw
    parts = [camera(H, W, (x, y, EGO_Z), s, 0.8 * W) for (x, y) in ((1.5, -40.0), (-2.0, 30.0)) for s in (1, -1)]
    parts += [lidar((0.0, -12.0, EGO_Z + 0.2), n_azim), axis_rays(rng, n_axis), boundary_rays(rng, n_boundary), roi_face_rays(rng, n_axis)]
    return tested(np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]))


def frame_rays():
    """one 1920 x 1280 camera frame (2.46 M rays) from inside the box, looking along +y"""
    return tested(*camera(1280, 1920, (0.5, -50.0, EGO_Z), 1, 2000.0))


def grid(kind, res, seed=0):
    """bool[X, Y, Z] in the normalised box: 'blocks' (a ground slab at the road plus random blocks on it), 'checker' (the most voxel
    transitions), 'full', 'empty', 'corner' (only the cell at x = +20, y = -75, z = -7.5 m, where the corner rays start)"""
    X, Y, Z = res
    g = np.zeros(res, dtype=bool)
    if kind == "blocks":
        rng = np.random.default_rng(seed)
        zc = ((np.arange(Z) + 0.5) / Z * 2 - 1) * HALF[2]
        g[:, :, np.abs(zc - (EGO_Z - 2.0)) < 1.0] = True
        z0 = int(np.argmax(np.abs(zc - (EGO_Z - 2.0)) < 1.0))
        for _ in range(60):
            sx, sy, sz = rng.integers(1, max(2, X // 6)), rng.integers(1, max(2, Y // 10)), rng.integers(1, max(2, Z // 2))
            x0, y0 = rng.integers(0, X - sx + 1), rng.integers(0, Y - sy + 1)
            g[x0:x0 + sx, y0:y0 + sy, z0:z0 + sz] = True
    elif kind == "checker":
        i, j, k = np.meshgrid(np.arange(X), np.arange(Y), np.arange(Z), indexing="ij")
        g = (i + j + k) % 2 == 0
    elif kind == "full":
        g[:] = True
    elif kind == "corner":
        g[X - 1, 0, 0] = True
    else:
        assert kind == "empty", kind
    return torch.from_numpy(np.ascontiguousarray(g))


# (name, grid kind, resolution, roi, dt_gamma, max_step_size, max_steps) of the single-grid march over street_rays()
SINGLE = [
    ("small_blocks", "blocks", SMALL, ROI, 0.0, 1e10, MAX_STEPS),
    ("small_blocks_gamma", "blocks", SMALL, ROI, 0.01, 1.0, MAX_STEPS),
    ("small_checker", "checker", SMALL, ROI, 0.0, 1e10, MAX_STEPS),
    ("small_full_cap", "full", SMALL, ROI, 0.0, 1e10, 256),
    ("small_empty", "empty", SMALL, ROI, 0.0, 1e10, MAX_STEPS),
    ("small_corner", "corner", SMALL, ROI, 0.0, 1e10, MAX_STEPS),
    ("roi_face_full", "full", SMALL, ROI_FACE, 0.0, 1e10, MAX_STEPS),
    ("large_blocks", "blocks", LARGE, ROI, 0.0, 1e10, MAX_STEPS),
    ("large_blocks_gamma", "blocks", LARGE, ROI, 0.02, 0.6, MAX_STEPS),
    ("large_checker", "checker", LARGE, ROI, 0.0, 1e10, MAX_STEPS),
    ("large_corner", "corner", LARGE, ROI, 0.0, 1e10, MAX_STEPS),
    ("smem_edge_blocks", "blocks", SMEM_EDGE, ROI, 0.0, 1e10, MAX_STEPS),
    ("global_edge_blocks", "blocks", GLOBAL_EDGE, ROI, 0.0, 1e10, MAX_STEPS),
]

# the batched march: five grids with distinct rois (batched_marching.cu: roi + 6 b, grid + b X Y Z)
BATCH_ROIS = ((-1., -1., -1., 1., 1., 1.), ROI_FACE, (-0.8, -1., -0.9, 1., 0.6, 0.7), (-1., -0.25, -1., 0.75, 1., 1.),
              (-0.5, -0.9, -1., 0.9, 0.9, 0.25))
BATCH_KINDS = ("blocks", "checker", "full", "corner", "blocks")


def batched_grid(res):
    return torch.stack([grid(k, res, seed=b) for b, k in enumerate(BATCH_KINDS)]).contiguous(), torch.tensor(BATCH_ROIS, dtype=torch.float32)
