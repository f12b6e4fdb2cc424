"""Learnable appearance codes on the cfg3 colour model (bench_cfg3.py: cuboid LoTD at 16 levels, 8192 camera rays per step, loss_cam),
one code per image for 8 images, gathered per ray (codes[image]) as the reference renderer does.  Arms, alternated in rounds in one
process, each timed with CUDA events around whole steps (forward + backward, ending in a device synchronise):
  host-module   the host-sized step with codes that require grad and the colour query on the module path -- what the parent commit ran
                for learnable codes (LoTDNeuS.forward -> autograd.grad -> half-precision RadianceNet)
  host-fused    the same step on the fused colour op with the code gradient (nsb_fused_color_bwd_appear)
  graph-off     StaticFrame with h_appear_grad=False (codes read, no code gradient)
  graph-on      StaticFrame with h_appear_grad=True
  graph-on+apply  the same, and the trainer's codes[image].backward(frame.d_h_appear) after each replay
Then k_color_rad_bwd<false> / <true> and k_ray_row_sum under torch.profiler (a separate run of host-sized steps with detached and
with learnable codes).  Prints one JSON line per round and a summary line with the GPU name, power limit and SM clocks read in the same run.

    python profiles/appear_grad_step.py --steps 20 --warmup 5 --rounds 3
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("appear_grad_step.py needs a CUDA device")
    import bench_cfg3 as C
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.renderer import SingleVolumeRenderer
    dev = torch.device("cuda:0")
    model = C.build_model(dev).train()
    n_img = 8
    batches = []
    for k in range(n_img):
        o, d = C.camera_rays(k, C.N_CAM)
        batches.append((o.to(dev), d.to(dev), torch.full((C.N_CAM,), k, dtype=torch.long, device=dev)))
    codes = torch.nn.Parameter(torch.randn(n_img, 4, generator=torch.Generator().manual_seed(0)).mul_(0.1).to(dev))
    renderer = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR)).train()
    color_fusable = type(model)._color_fusable

    def host_step(b, fused):
        o, d, img = b
        model.zero_grad(set_to_none=False)
        codes.grad = None
        model._color_fusable = (lambda: color_fusable(model)) if fused else (lambda: False)
        out = renderer.render(model, o, d, rays_h_appear=codes[img])["rendered"]
        C.loss_cam(out).backward()

    frames = {}
    for on in (False, True):
        f = StaticFrame(model, C.N_CAM, loss_fn=C.loss_cam, near=C.NEAR, far=C.FAR, slack=2.0, zero_grads=True, h_appear_grad=on)
        for o, d, _ in batches:
            f.rays_o.copy_(o); f.rays_d.copy_(d); f._size()
        frames[on] = f

    def graph_step(b, on, apply=False):
        o, d, img = b
        ha = codes[img]
        frames[on].step(o, d, ha.detach())
        if apply:
            codes.grad = None
            ha.backward(frames[on].d_h_appear)

    arms = {"host-module": lambda b: host_step(b, False), "host-fused": lambda b: host_step(b, True),
            "graph-off": lambda b: graph_step(b, False), "graph-on": lambda b: graph_step(b, True),
            "graph-on+apply": lambda b: graph_step(b, True, True)}
    for name, fn in arms.items():                                   # warm every arm (capture, allocator) before any timing
        for s in range(args.warmup):
            fn(batches[s % n_img])
    torch.cuda.synchronize()
    for f in frames.values():
        assert f.counts()["overflow"] == 0
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
    # kernel times of the radiance backward with and without the code gradient
    from torch.profiler import ProfilerActivity, profile
    kern = {}
    for label, learn in (("detached-codes", False), ("learnable-codes", True)):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for s in range(args.steps):
                o, d, img = batches[s % n_img]
                model.zero_grad(set_to_none=False)
                model._color_fusable = lambda: color_fusable(model)
                ha = codes[img] if learn else codes[img].detach()
                C.loss_cam(renderer.render(model, o, d, rays_h_appear=ha)["rendered"]).backward()
            torch.cuda.synchronize()
        for e in prof.key_averages():
            if "k_color_rad_bwd" in e.key or "k_ray_row_sum" in e.key:
                kern[f"{label}: {e.key.split('(')[0]}"] = dict(calls=e.count, us_per_call=round(e.device_time_total / max(e.count, 1), 1))
    print(json.dumps(dict(summary={k: dict(median_ms=round(statistics.median(v), 3), min_ms=round(min(v), 3)) for k, v in times.items()},
                          kernels=kern, steps=args.steps, rounds=args.rounds, rays=C.N_CAM, gpu=gpu_info(),
                          torch=torch.__version__)), flush=True)


if __name__ == "__main__":
    main()
