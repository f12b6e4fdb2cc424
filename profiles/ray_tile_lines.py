"""Distinct 128-byte table lines per gather instruction of the ray-tiled SDF query (k_fused_sdf_tc, mode 2) for the tile shapes a warp's
32 rays can take in the image, counted on the CPU with the kernel's own addressing (oracle/lotd.py: pos_fract with scale = res - 2,
grid_index: dense strides or the hash and `% size`, 2 fp16 features = 4 bytes per cell).

Workload: the bench model's table geometry (16 levels, gen_ngp, 2^19 hash entries), all 8 bench views of 800 x 600, the rays that pass
the box test.  Every ray has the 65 linear coarse samples; the rays that the occupancy grid marcher (oracle/march.py) finds occupied
voxels on also have 51 fine samples, merged in depth order as in the boundary query.  The fine samples themselves come from the
up-sampling, which this script does not run: they are placed evenly over the ray's marched interval (where the up-sampling puts them,
near the surface), so the fine-sample lines are an estimate; the coarse-sample lines and the idle lanes are exact.

Mode 2 walks the packs in groups of 32 (lane = ray) and, per group, sample ordinal k of all 32 rays in one gather per corner and level.
A tile shape tw x th groups the packs by (py / th, px / tw, (py % th) tw + px % tw); 32 x 1 is the image-row order.  Reported per shape:
distinct lines per group and gather ordinal, per level and in sum over the 16 levels (all 8 corners of one level count as one set, the
lines the L1 tag stage sees for one level of one sample ordinal), and the mean idle lane-samples per group (sum of max_n - n over lanes).

    python profiles/ray_tile_lines.py [--every 4] [--views 8]
"""
import argparse
import json
import os
import sys
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import lotd as olotd, march as omarch, render as orender, scene as oscene  # noqa: E402

H, W, N_VIEWS = 600, 800, 8
N_COARSE1, N_FINE = 65, 51
SHAPES = ((32, 1), (16, 2), (8, 4), (4, 8))


def tile_perm(py, px, tw, th):
    return np.lexsort(((py % th) * tw + px % tw, px // tw, py // th))


def view_counts(k, every):
    meta = olotd.LoDMeta(3, **olotd.gen_ngp_cfg())
    ro, rd = oscene.pinhole_rays(H, W, oscene.orbit_camera(k, N_VIEWS))
    rt = orender.ray_test(ro, rd, near=0.01)
    inds = rt["rays_inds"].numpy()
    o, d = rt["rays_o"].numpy().astype(np.float32), rt["rays_d"].numpy().astype(np.float32)
    near, far = rt["near"], rt["far"]
    n = inds.shape[0]
    coarse = orender.batch_sample_step_linear(near, far, N_COARSE1)[0].numpy().astype(np.float32)
    info, t0 = omarch.ray_marching(rt["rays_o"], rt["rays_d"], near, far, torch.tensor([-1., -1, -1, 1, 1, 1]), oscene.make_occ_grid(), 0.005, 1e10,
                                   0.0, 4096)[:2]
    info, t0 = info.numpy(), t0.numpy()
    hit = info[:, 1] > 0
    cnt = np.where(hit, N_COARSE1 + N_FINE, N_COARSE1)
    t = np.full((n, N_COARSE1 + N_FINE), np.inf, dtype=np.float32)
    t[:, :N_COARSE1] = coarse
    h = np.nonzero(hit)[0]
    lo, hi = t0[info[h, 0]], t0[info[h, 0] + info[h, 1] - 1]
    t[h, N_COARSE1:] = lo[:, None] + (hi - lo)[:, None] * ((np.arange(N_FINE, dtype=np.float32) + 0.5) / N_FINE)[None, :]
    t.sort(axis=1)
    py, px = inds // W, inds % W
    perms = {f"{tw}x{th}": tile_perm(py, px, tw, th) for tw, th in SHAPES}
    n_groups = (n + 31) // 32
    pad = n_groups * 32 - n
    lines = {s: np.zeros(meta.n_levels) for s in perms}
    gathers = {s: 0 for s in perms}
    idle = {}
    for s, p in perms.items():
        c = np.concatenate([cnt[p], np.zeros(pad, dtype=cnt.dtype)]).reshape(n_groups, 32)
        idle[s] = float((c.max(1, keepdims=True) - c).sum() / n_groups)
    ords = list(range(0, N_COARSE1 + N_FINE, every))
    for j in ords:
        valid = j < cnt
        x = o + d * np.where(valid, t[:, j], 0.)[:, None]
        x = np.clip(x * np.float32(0.5) + np.float32(0.5), 1e-6, 1 - 1e-6).astype(np.float32)
        for lvl in range(meta.n_levels):
            res = np.array(meta.level_res_multidim[lvl], dtype=np.uint32)
            cell, _ = olotd.pos_fract(x, (res - 2).astype(np.float32))
            nf = meta.level_n_feats[lvl]
            ln = np.stack([(meta.level_offsets[lvl] + olotd.grid_index(meta, lvl, cell + off) * nf) * 2 // 128
                           for _, off, _ in olotd._corner_weights(np.zeros((1, 3), np.float32), 3)], 1)
            ln[~valid] = -1
            for s, p in perms.items():
                g = np.concatenate([ln[p], np.full((pad, 8), -1, dtype=ln.dtype)]).reshape(n_groups, 256)
                g.sort(axis=1)
                distinct = (np.diff(g, axis=1) != 0).sum(1) + 1 - (g[:, 0] == -1)
                active = g[:, -1] != -1                  # groups with a lane at this ordinal issue the gather
                lines[s][lvl] += distinct[active].sum()
                if lvl == 0:
                    gathers[s] += int(active.sum())
    return dict(view=k, rays=int(n), hit=int(hit.sum()), lines={s: lines[s].tolist() for s in perms}, gathers=gathers, idle=idle, groups=n_groups)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--every", type=int, default=4, help="count every k-th sample ordinal (the ordinals are similar; 1 = all)")
    ap.add_argument("--views", type=int, default=N_VIEWS)
    args = ap.parse_args()
    with ProcessPoolExecutor(max_workers=min(args.views, os.cpu_count() or 1)) as ex:
        res = list(ex.map(view_counts, range(args.views), [args.every] * args.views))
    out = dict(rays=sum(r["rays"] for r in res), hit_rays=sum(r["hit"] for r in res), every=args.every, views=args.views, shapes={})
    for tw, th in SHAPES:
        s = f"{tw}x{th}"
        per_level = np.sum([r["lines"][s] for r in res], 0) / sum(r["gathers"][s] for r in res)
        out["shapes"][s] = dict(lines_per_gather=round(float(per_level.sum()), 1), per_level=[round(float(v), 2) for v in per_level],
                                idle_lane_samples_per_group=round(sum(r["idle"][s] * r["groups"] for r in res) / sum(r["groups"] for r in res), 1))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
