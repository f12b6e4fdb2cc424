"""Learnable rays (pose refinement) on the cfg3 colour model (bench_cfg3.py: cuboid LoTD at 16 levels): per step 8192 camera rays
(loss_cam, learnable appearance codes, one per image for 8 images) and 8192 LiDAR rays (loss_lidar, with_rgb=False), both built from a
learnable SE(3) pose correction, as the shipped configurations train from iteration 500 on.  Arms, alternated in rounds in one process,
each timed with CUDA events around whole steps (forward + backward, ending in a device synchronise):
  host-parent   the host-sized step with the selection the parent commit made for rays that require grad: the general query chain,
                the boundary SDF and the colour / normal query on the module path (no-grad march and up-sampling stay fused)
  host-fused    the same step on the fused query with the ray gradient (nsb_fused_sdf_bwd_rays, nsb_fused_color_bwd_grads)
  host-fixed    the fused step with a pose that needs no grad (the same rays, detached): the cost of the ray gradient itself
  graph         the one-launch graph step: one StaticFrame for the camera rays (h_appear_grad=True, ray_grad=True) and one for the LiDAR
                rays (with_rgb=False, ray_grad=True), replayed on the posed rays; the trainer's backward of the codes and of the pose
                (torch.autograd.backward of the rays with frame.d_rays_o / d_rays_d) runs outside the graphs
  graph-fixed   the same frames without ray_grad, the pose held fixed (the codes still get their gradient)
Prints one JSON line per round and a summary line with the GPU name, power limit and SM clocks read in the same run.

    python profiles/ray_grad_step.py --steps 20 --warmup 5 --rounds 3
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def pose(params, o, d):
    """rays under a small SE(3) correction: rotation exp(omega) (Rodrigues) about the ray origin's frame, then translation"""
    omega, trans = params[:3], params[3:]
    th = omega.norm().clamp_min(1e-12)
    k = omega / th
    z = torch.zeros((), device=o.device)
    K = torch.stack([torch.stack([z, -k[2], k[1]]), torch.stack([k[2], z, -k[0]]), torch.stack([-k[1], k[0], z])])
    R = torch.eye(3, device=o.device) + torch.sin(th) * K + (1 - torch.cos(th)) * (K @ K)
    return o @ R.T + trans, d @ R.T


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ray_grad_step.py needs a CUDA device")
    import bench_cfg3 as C
    from neuralsim_b200.graphics import neus as GN
    from neuralsim_b200.renderer import SingleVolumeRenderer
    dev = torch.device("cuda:0")
    model = C.build_model(dev).train()
    n_img = 8
    batches = []
    for k in range(n_img):
        (co, cd), (lo, ld) = C.make_views(k)
        batches.append((co.to(dev), cd.to(dev), lo.to(dev), ld.to(dev), torch.full((C.N_CAM,), k, dtype=torch.long, device=dev)))
    codes = torch.nn.Parameter(torch.randn(n_img, 4, generator=torch.Generator().manual_seed(0)).mul_(0.1).to(dev))
    params = torch.nn.Parameter(torch.tensor([1e-3, -2e-3, 1e-3, 0.02, -0.01, 0.01], device=dev))
    r_cam = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR)).train()
    r_lidar = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True)).train()
    orig = dict(qf=GN._query_fused, sdf_on_rays=type(model).forward_sdf_on_rays, color=type(model)._color_fusable, geo=type(model)._geometry_fusable)

    def select(parent):
        """the parent's choices for rays that require grad, or this commit's"""
        if parent:
            GN._query_fused = lambda *a, **k: None

            def sdf_on_rays(ridx, t, rays_o, rays_d, packs=None):
                if torch.is_grad_enabled():
                    return model.forward_sdf(torch.addcmul(rays_o[ridx], rays_d[ridx], t.unsqueeze(-1)))
                return orig["sdf_on_rays"](model, ridx, t, rays_o, rays_d, packs=packs)
            model.forward_sdf_on_rays = sdf_on_rays
            model._color_fusable = model._geometry_fusable = lambda: False
        else:
            GN._query_fused = orig["qf"]
            for k in ("forward_sdf_on_rays", "_color_fusable", "_geometry_fusable"):
                model.__dict__.pop(k, None)

    def host_step(b, parent, learnable=True):
        co, cd, lo, ld, img = b
        select(parent)
        model.zero_grad(set_to_none=False)
        codes.grad = params.grad = None
        p = params if learnable else params.detach()
        o1, d1 = pose(p, co, cd)
        o2, d2 = pose(p, lo, ld)
        loss = C.loss_cam(r_cam.render(model, o1, d1, rays_h_appear=codes[img])["rendered"]) + C.loss_lidar(r_lidar.render(model, o2, d2)["rendered"])
        loss.backward()

    # the graph step: per arm a camera frame (zeroes the gradients in its graph) and a LiDAR frame (adds to them), sized on every batch
    from neuralsim_b200.graphics.neus_static import StaticFrame
    frames = {}
    for learn in (True, False):
        fc = StaticFrame(model, C.N_CAM, loss_fn=C.loss_cam, near=C.NEAR, far=C.FAR, slack=2.0, zero_grads=True, h_appear_grad=True, ray_grad=learn)
        fl = StaticFrame(model, C.N_LIDAR, loss_fn=C.loss_lidar, near=C.NEAR, far=C.FAR, with_rgb=False, slack=2.0, ray_grad=learn)
        with torch.no_grad():
            for co, cd, lo, ld, _ in batches:
                for f, (o, d) in ((fc, pose(params, co, cd)), (fl, pose(params, lo, ld))):
                    f.rays_o.copy_(o); f.rays_d.copy_(d); f._size()
        frames[learn] = (fc, fl)

    def graph_step(b, learnable):
        co, cd, lo, ld, img = b
        select(False)
        codes.grad = params.grad = None
        fc, fl = frames[learnable]
        p = params if learnable else params.detach()
        o1, d1 = pose(p, co, cd)
        o2, d2 = pose(p, lo, ld)
        ha = codes[img]
        fc.step(o1.detach(), d1.detach(), ha.detach())
        fl.step(o2.detach(), d2.detach())
        if learnable:
            torch.autograd.backward([ha, o1, d1, o2, d2], [fc.d_h_appear, fc.d_rays_o, fc.d_rays_d, fl.d_rays_o, fl.d_rays_d])
        else:
            ha.backward(fc.d_h_appear)

    arms = {"host-parent": lambda b: host_step(b, True), "host-fused": lambda b: host_step(b, False),
            "host-fixed": lambda b: host_step(b, False, learnable=False), "graph": lambda b: graph_step(b, True),
            "graph-fixed": lambda b: graph_step(b, False)}
    for name, fn in arms.items():
        for s in range(args.warmup):
            fn(batches[s % n_img])
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for r in range(args.rounds):
        order = list(arms) if r % 2 == 0 else list(reversed(list(arms)))
        line = {"round": r}
        for name in order:
            fn = arms[name]
            for s in range(args.warmup):
                fn(batches[s % n_img])
            ms = []
            for s in range(args.steps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                a.record()
                fn(batches[s % n_img])
                b.record()
                torch.cuda.synchronize()
                ms.append(a.elapsed_time(b))
            times[name] += ms
            line[name] = round(statistics.median(ms), 3)
        print(json.dumps(line), flush=True)
    select(False)
    print(json.dumps(dict(summary={k: dict(median_ms=round(statistics.median(v), 3), min_ms=round(min(v), 3)) for k, v in times.items()},
                          steps=args.steps, rounds=args.rounds, rays=dict(camera=C.N_CAM, lidar=C.N_LIDAR), gpu=gpu_info(),
                          torch=torch.__version__)), flush=True)


if __name__ == "__main__":
    main()
