"""The LiDAR batch drawn inside the one-launch step: what it costs and saves.  Arms, alternated in rounds in one process, each timed with
CUDA events around whole steps (draw + forward + LidarLoss + backward):
  graph_sampler  StaticFrame(sampler=LidarSampler(...), perturb=True): one graph launch draws the frame's merged_weighted batch, moves the
                 beams to world, renders and takes the loss (csrc/lidar_sample.cu)
  graph_recipe   the same graph step fed by the reference's torch ops: recipe_sample_merged (unique_consecutive, the .cpu() read, the numpy
                 split, one randint per lidar, the gathers), the world transform as MultiRaysLidarBundle.get_selected_rays computes it
                 ((R * x).sum(-1) + t), LidarLoss.set_step copying the ranges, then frame.step(rays_o, rays_d)
Workload: the shipped 12-level LiDAR-only model (profiles/lidar_only_shipped_step.py) on the cfg3 street, 8192 rays per step, the shipped
lidar_weight [0.4, 0.1, 0.1, 0.1, 0.1], 5 lidars with Waymo-like beam counts (a ~150 k-beam top lidar and four of ~4 k, one of them
missing in some frames), 20 frames, a new frame every step.  Prints one JSON line per round and a summary line with the GPU name, power
limit and SM clocks read in the same run; `--out FILE` also writes the summary there.

    python profiles/lidar_sampler_step.py --steps 20 --warmup 5 --rounds 4
"""
import argparse
import gc
import json
import math
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

N, FRAMES = 8192, 20
WEIGHT = [0.4, 0.1, 0.1, 0.1, 0.1]
LIDAR_CFG = dict(discard_outliers=0, discard_outliers_median=100.0, discard_toofar=80.0, depth=dict(w=0.05, fn_type="l1"),
                 line_of_sight=dict(w=0.1, fn_type="neus_unisim", fn_param=dict(epsilon_anneal=dict(type="milestones", milestones=[5000, 10000],
                                                                                                     vals=[1.5, 0.75, 0.5]))))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def data(dev, seed=0):
    """FRAMES frames of 5 lidars driving along the street: lidar-local beams, ranges to the road plane, per-frame lidar-to-world transforms"""
    import bench_cfg3 as C
    g = np.random.default_rng(seed)
    mounts = [(0.0, 0.0, 2.2, 0.0), (1.5, 1.0, 0.8, 0.6), (1.5, -1.0, 0.8, -0.6), (-2.0, 0.7, 0.9, 2.5), (-2.0, -0.7, 0.9, -2.5)]
    counts = np.stack([g.integers(140000, 160000, FRAMES)] + [g.integers(3000, 5000, FRAMES) for _ in range(4)], 1)
    counts[::7, 2] = 0
    l2w = np.zeros((FRAMES, 5, 3, 4))
    os_, ds, rs = [], [], []
    for f in range(FRAMES):
        for li, n in enumerate(counts[f]):
            mx, my, mz, yaw = mounts[li]
            c, s = math.cos(yaw), math.sin(yaw)
            R, t = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]), np.array([mx, my - 60.0 + 6.0 * f, mz + C.ROAD_Z])
            l2w[f, li, :, :3], l2w[f, li, :, 3] = R, t
            elev, azim = np.radians(g.uniform(-17.6, 2.4, n)), g.uniform(0, 2 * math.pi, n)
            d = np.stack([np.cos(elev) * np.sin(azim), np.cos(elev) * np.cos(azim), np.sin(elev)], -1)
            dz = (d @ R.T)[:, 2]
            r = np.where(dz < -1e-3, (C.ROAD_Z - t[2]) / np.where(dz < -1e-3, dz, -1.0), 0.0)
            os_.append(np.zeros((n, 3), np.float32)), ds.append(d.astype(np.float32)), rs.append(np.clip(r, 0, 150).astype(np.float32))
    cat = lambda v: torch.from_numpy(np.concatenate(v)).to(dev).contiguous()
    return cat(os_), cat(ds), cat(rs), counts, torch.from_numpy(l2w.astype(np.float32)).to(dev).contiguous()


def timed(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lidar_sampler_step.py: no CUDA device")
    import bench_cfg3 as C
    from lidar_only_shipped_step import _model
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.lidar_sampler import LidarSampler
    from neuralsim_b200.loss import LidarLoss
    dev = torch.device("cuda")
    model = _model(dev)
    o, d, r, counts, l2w = data(dev)
    s = LidarSampler(o, d, r, counts, l2w, N, multi_lidar_weight=WEIGHT)
    it = [0]

    la, lb = LidarLoss(**LIDAR_CFG), LidarLoss(**LIDAR_CFG)
    model.zero_grad(set_to_none=True)
    gc.collect()
    fa = StaticFrame(model, N, loss_fn=lambda ret, gt: sum(la(None, ret, ground_truth=gt).values()), loss_on_ret=True, near=C.NEAR, far=C.FAR,
                     with_rgb=False, zero_grads=True, perturb=True, sampler=s)
    fb = StaticFrame(model, N, loss_fn=lambda ret: sum(lb(None, ret).values()), loss_on_ret=True, near=C.NEAR, far=C.FAR, with_rgb=False,
                     zero_grads=True, perturb=True)

    def step_sampler():
        f = it[0] % FRAMES
        it[0] += 1
        la.set_step(None, it[0])
        fa.step(frame_ind=f)

    def step_recipe():
        f = it[0] % FRAMES
        it[0] += 1
        b = s.recipe(f)
        T = l2w[f][b["li"]]
        R, t = T[..., :3], T[..., 3]
        ro, rd = (R * b["rays_o"].unsqueeze(-2)).sum(-1) + t, (R * b["rays_d"].unsqueeze(-2)).sum(-1)
        lb.set_step(b["ranges"], it[0])
        fb.step(ro, rd)

    arms = dict(graph_sampler=step_sampler, graph_recipe=step_recipe)
    for fn in arms.values():
        for _ in range(a.warmup):
            fn()
    for fr in (fa, fb):
        fr.check()
    res = {k: [] for k in arms}
    for rnd in range(a.rounds):
        order = list(arms) if rnd % 2 == 0 else list(arms)[::-1]
        line = {}
        for k in order:
            line[k] = timed(arms[k], a.steps)
            res[k].append(line[k])
        print(json.dumps(dict(round=rnd, ms_per_step=line)))
    summary = dict(workload=f"12-level LiDAR-only model, {N} LiDAR rays per step, 5 lidars, {FRAMES} frames, perturbed",
                   gpu=gpu_info(), median_ms_per_step={k: statistics.median(v) for k, v in res.items()},
                   overflow=[fr.counts()["overflow"] for fr in (fa, fb)], captures=[fa.captures, fb.captures])
    print(json.dumps(summary))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(summary, fh, indent=1)


if __name__ == "__main__":
    main()
