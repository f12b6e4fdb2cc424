"""Error-map importance sampling in the one-launch step: what drawing the batch inside the graph costs and saves.  Arms, alternated in
rounds in one process, each timed with CUDA events around whole steps (sample + forward + loss + backward + error-map update):
  graph_sampler  StaticFrame(pose=..., perturb=True, sampler=CameraSampler(...)): one graph launch draws frames and pixels, gathers the
                 ground truth, renders, and updates the error map (csrc/importance.cu)
  graph_eager    the same graph step without the sampler, fed by the reference's recipe: ImpSampler.sample_img_pixel's torch ops, fi.cpu()
                 (the host round trip of JointFramePixelDataset.sample), the ground truth gathered on the CPU and copied to the device,
                 the pixels lifted with torch ops, frame.step(dirs=..., pidx=...), then ErrorMap.update_error_map's torch ops
Workload: the cfg3 street model (bench_cfg3.build_model, 16 levels), one 960 x 640 camera of 40 frames, 8192 rays per step, a learnable
pose, perturbed samples, error_map_hw (32, 64), frac_uniform 0.5.  A third measurement times the sampler and update kernels alone against
the same torch ops captured in one CUDA graph (`kernels` / `torch_graph`, ms per batch).  Prints one JSON line per round and a summary
line with the GPU name, power limit and SM clocks read in the same run; `--out FILE` also writes the summary there.

    python profiles/error_map_step.py --steps 20 --warmup 5 --rounds 4
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

F, W, H, FOCAL, N = 40, 960, 640, 1000.0, 8192


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def camera(dev):
    from neuralsim_b200 import importance as I
    g = torch.Generator(dev).manual_seed(0)
    m = I.ErrorMap(F, (32, 64), n_steps_max=500, device=dev)
    m.error_map.copy_(torch.rand(m.error_map.shape, device=dev, generator=g))
    m.construct_cdf()
    s = I.ImpSampler({"rgb": (m, 0.5)}, frac_uniform=0.5)
    gts = dict(image_rgb=torch.rand(F, H, W, 3, device=dev, generator=g), image_occupancy_mask=torch.rand(F, H, W, device=dev, generator=g) > 0.1)
    K = torch.tensor([[FOCAL, 0, W / 2], [0, FOCAL, H / 2], [0, 0, 1]], dtype=torch.float32).repeat(F, 1, 1).to(dev).contiguous()
    return I.CameraSampler([s], [gts], [K], [(W, H)], pose_bases=[0]), s


def loss_fn(rendered, gt):
    diff = (rendered["rgb_volume"] - gt["image_rgb"]).abs()
    return diff.mean(), diff.mean(-1) * gt["image_occupancy_mask"].float()


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
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("error_map_step.py needs a CUDA device")
    import bench_cfg3 as C
    import pose64
    from neuralsim_b200 import importance as I
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.graphics.pose import CameraPoses
    dev = torch.device("cuda:0")
    model = C.build_model(dev).train()
    q0, t0 = pose64.street_poses(1, F, C.ROAD_Z)
    poses = CameraPoses(torch.as_tensor(q0, dtype=torch.float32), torch.as_tensor(t0, dtype=torch.float32)).to(dev)
    cs, samp = camera(dev)
    em = samp.error_map
    gt_cpu = {k: v.cpu() for k, v in cs.gts[0].items()}
    gc.collect()
    fr_s = StaticFrame(model, N, loss_fn=loss_fn, near=C.NEAR, far=C.FAR, zero_grads=True, slack=2.0, pose=poses, perturb=True, sampler=cs)
    # the eager arm: the graph step reads its ground truth from static buffers, and leaves the per-ray error in one
    gt_dev = {k: torch.zeros((N,) + tuple(v.shape[3:]), dtype=v.dtype, device=dev) for k, v in cs.gts[0].items()}
    err_dev = torch.zeros(N, device=dev)

    def eager_loss(rendered):
        loss, err = loss_fn(rendered, gt_dev)
        err_dev.copy_(err.detach())
        return loss
    fr_e = StaticFrame(model, N, loss_fn=eager_loss, near=C.NEAR, far=C.FAR, zero_grads=True, slack=2.0, pose=poses, perturb=True)
    wh = torch.tensor([W, H], device=dev)

    def eager_step():
        fi, xy = I.recipe_sample_img_pixel((em.cdf_x_cond_y, em.cdf_y, em.cdf_img), F, N, 0.5)
        fi_c = fi.cpu()                                               # JointFramePixelDataset.sample: fi.cpu(), the gather on the host
        w, h, dirs = I.recipe_pixels(xy, fi, wh, cs.intrs[0])
        w_c, h_c = w.cpu(), h.cpu()
        for k, v in gt_cpu.items():
            gt_dev[k].copy_(v[fi_c, h_c, w_c], non_blocking=False)
        fr_e.step(dirs=dirs, pidx=fi)
        I.recipe_update_error_map(em.error_map, fi, xy, err_dev)
        em.count_step()

    arms = dict(graph_sampler=lambda: fr_s.step(cam=0), graph_eager=eager_step)
    for fn in arms.values():
        for _ in range(args.warmup):
            fn()
    assert fr_s.check(retry=False) and fr_e.check(retry=False), "arena overflow after the warm-up"
    res = {k: [] for k in arms}
    for r in range(args.rounds):
        line = {}
        order = list(arms.items())
        for k, fn in (order if r % 2 == 0 else order[::-1]):
            line[k] = timed(fn, args.steps)
            res[k].append(line[k])
        print(json.dumps(dict(workload="cfg3 street 8192 camera rays", round=r, ms_per_step=line)), flush=True)
    # ---- the sampler and update alone: the kernels against the same torch ops captured in a CUDA graph
    fidx, xy = torch.zeros(N, dtype=torch.int64, device=dev), torch.zeros(N, 2, device=dev)
    pidx, dirs = torch.zeros(N, dtype=torch.int64, device=dev), torch.zeros(N, 3, device=dev)
    gts = {k: torch.zeros_like(v) for k, v in gt_dev.items()}
    cam = torch.zeros((), dtype=torch.int64, device=dev)
    rng, flag = torch.zeros(2, dtype=torch.int64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
    err = torch.rand(N, device=dev)

    def kernels():
        cs.sample(cam, rng, N, fidx, xy, pidx, dirs, gts, None, None)
        cs.update(cam, fidx, xy, err, flag)

    def torch_ops():
        fi, pxy = I.recipe_sample_img_pixel((em.cdf_x_cond_y, em.cdf_y, em.cdf_img), F, N, 0.5)
        w, h, d = I.recipe_pixels(pxy, fi, wh, cs.intrs[0])
        for k, v in cs.gts[0].items():
            gts[k].copy_(v[fi, h, w])
        dirs.copy_(d)
        I.recipe_update_error_map(em.error_map, fi, pxy, err)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            torch_ops()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        torch_ops()
    for _ in range(args.warmup):
        kernels()
        g.replay()
    parts = dict(kernels=[], torch_graph=[])
    for r in range(args.rounds):
        parts["kernels"].append(timed(kernels, 200))
        parts["torch_graph"].append(timed(g.replay, 200))
    out = dict(workload="cfg3 street 8192 camera rays, pose + perturb", rays=N, camera=[F, W, H], captures=fr_s.captures,
               median_ms=({k: statistics.median(v) for k, v in res.items()}), sampler_update_ms={k: statistics.median(v) for k, v in parts.items()},
               gpu=gpu_info())
    print(json.dumps(out), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
