"""Camera-pose refinement in the one-launch step: the trainer's current recipe against the pose inside the graph.  Arms, alternated in
rounds in one process, each timed with CUDA events around whole steps (forward + backward of the rays, the pose and the model):
  recipe   the reference's pose arithmetic in torch (tests/pose64.py torch_pose_rays: normalize_quat, quat_apply, normalize), the rays
           copied into StaticFrame(ray_grad=True), one replay, then torch.autograd.backward through the pose with frame.d_rays_o / d_rays_d
  graph    StaticFrame(pose=CameraPoses(...)): the pose's rays (nsb_pose_rays) and its adjoint (nsb_pose_rays_backward) inside the graph,
           one replay, the gradient in dq.grad / dt.grad
Workloads: the cfg3 street model (bench_cfg3.build_model, 16 levels) with 8192 camera rays over 3 cameras x 8 frames per step (a new
random batch of pixels and poses each step), and bench.py's model at its 800 x 600 frame (one pose).  Prints one JSON line per round and
workload and a summary line with the GPU name, power limit and SM clocks read in the same run.

    python profiles/pose_refine_step.py --steps 20 --warmup 5 --rounds 3
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
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def street(dev, n_batches):
    import bench_cfg3 as C
    import pose64
    model = C.build_model(dev).train()
    q0, t0 = pose64.street_poses(3, 8, C.ROAD_Z)
    batches = []
    for k in range(n_batches):
        pidx, dirs = pose64.street_batch(C.N_CAM, 24, seed=100 + k)
        batches.append((torch.from_numpy(pidx).to(dev), torch.from_numpy(dirs).to(dev)))
    return model, q0, t0, batches, C.loss_cam, dict(near=C.NEAR, far=C.FAR)


def frame800(dev):
    import bench
    import pose64
    from oracle import scene as oscene
    model = bench.build_model(dev).train()
    cam = np.array(oscene.orbit_camera(0, bench.N_VIEWS))
    fwd = -cam / np.linalg.norm(cam)
    right = np.cross(fwd, [0.0, 0.0, 1.0])
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    q0 = pose64.rot_to_quat(np.stack([right, down, fwd], 1))[None].astype(np.float32)
    H, W = bench.H, bench.W
    f = (H + W) / 2.0
    j, i = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    dirs = np.stack([(i.ravel() + 0.5 - W / 2) / f, (j.ravel() + 0.5 - H / 2) / f, np.ones(H * W)], -1).astype(np.float32)
    batch = (torch.zeros(H * W, dtype=torch.int64, device=dev), torch.from_numpy(dirs).to(dev))
    return model, q0, cam[None].astype(np.float32), [batch], bench.loss_of, dict(near=0.01)


def run(name, make, dev, args):
    import pose64
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.graphics.pose import CameraPoses
    model, q0, t0, batches, loss, cfg = make()
    n = batches[0][1].shape[0]
    poses = CameraPoses(torch.from_numpy(q0), torch.from_numpy(t0)).to(dev)
    with torch.no_grad():
        poses.dq.normal_(0.0, 1e-3)
    gc.collect()
    fr_new = StaticFrame(model, n, loss_fn=loss, zero_grads=True, pose=poses, slack=2.0, **cfg)
    fr_old = StaticFrame(model, n, loss_fn=loss, zero_grads=True, ray_grad=True, slack=2.0, **cfg)

    def step_recipe(b):
        poses.dq.grad = poses.dt.grad = None
        o, d = pose64.torch_pose_rays(poses.q0, poses.dq, poses.t0, poses.dt, b[0], b[1])
        fr_old.step(o.detach(), d.detach())
        torch.autograd.backward([o, d], [fr_old.d_rays_o, fr_old.d_rays_d])

    def step_graph(b):
        poses.dq.grad = poses.dt.grad = None
        fr_new.step(dirs=b[1], pidx=b[0])

    arms = dict(recipe=step_recipe, graph=step_graph)
    for fn in arms.values():
        for k in range(args.warmup):
            fn(batches[k % len(batches)])
    torch.cuda.synchronize()
    res = {k: [] for k in arms}
    for r in range(args.rounds):
        line = {}
        for k, fn in (arms.items() if r % 2 == 0 else reversed(list(arms.items()))):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            for s in range(args.steps):
                fn(batches[s % len(batches)])
            b.record()
            torch.cuda.synchronize()
            line[k] = a.elapsed_time(b) / args.steps
            res[k].append(line[k])
        print(json.dumps(dict(workload=name, round=r, ms_per_step=line)), flush=True)
    out = dict(workload=name, rays=n, poses=int(q0.shape[0]), captures=dict(graph=fr_new.captures, recipe=fr_old.captures),
               median_ms={k: statistics.median(v) for k, v in res.items()})
    del fr_new, fr_old
    gc.collect()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--only", choices=["street", "frame800"], default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pose_refine_step.py needs a CUDA device")
    dev = torch.device("cuda:0")
    out = []
    if args.only in (None, "street"):
        out.append(run("cfg3 street 8192 rays, 3 cameras x 8 frames", lambda: street(dev, 8), dev, args))
    if args.only in (None, "frame800"):
        out.append(run("800x600 frame, one pose", lambda: frame800(dev), dev, args))
    print(json.dumps(dict(summary=out, gpu=gpu_info())), flush=True)


if __name__ == "__main__":
    main()
