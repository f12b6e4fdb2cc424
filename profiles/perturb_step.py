"""Perturbed samples in the one-launch step: what drawing torch's random stream inside the graph costs.  Arms, alternated in rounds in
one process, each timed with CUDA events around whole steps (forward + loss + backward):
  graph          StaticFrame(perturb=False): the unperturbed graph step (below 8192 tested rays it runs the persistent up-sampling kernel)
  graph_perturb  StaticFrame(perturb=True): the coarse depths and the stage quantiles drawn in csrc/perturb.cu (the stage kernels, never
                 the persistent kernel -- as on the host-sized path)
  host_perturb   SingleVolumeRenderer(perturb=True).render + backward: the host-sized perturbed step (torch.rand, three host reads)
Workloads: the cfg3 street model (bench_cfg3.build_model, 16 levels) with 8192 camera rays and with 8192 LiDAR rays, and bench.py's
model at its 800 x 600 frame.  Prints one JSON line per round and workload and a summary line with the GPU name, power limit and SM
clocks read in the same run; `--out FILE` also writes the summary there.

    python profiles/perturb_step.py --steps 20 --warmup 5 --rounds 4
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def street(dev, lidar):
    import bench_cfg3 as C
    model = C.build_model(dev).train()
    if lidar:
        o, d = C.lidar_rays(1, C.N_LIDAR)
        return model, o.to(dev), d.to(dev), None, C.loss_lidar, dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True)
    o, d = C.camera_rays(3, C.N_CAM)
    return model, o.to(dev), d.to(dev), torch.zeros(o.shape[0], 4, device=dev), C.loss_cam, dict(near=C.NEAR, far=C.FAR)


def frame800(dev):
    import bench
    from oracle import scene as oscene
    model = bench.build_model(dev).train()
    o, d = oscene.pinhole_rays(bench.H, bench.W, oscene.orbit_camera(0, bench.N_VIEWS))
    return model, o.to(dev), d.to(dev), torch.zeros(o.shape[0], 4, device=dev), bench.loss_of, dict(near=0.01)


def run(name, make, args):
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.renderer import SingleVolumeRenderer
    model, o, d, codes, loss, cfg = make()
    n = o.shape[0]
    gc.collect()
    frames = {k: StaticFrame(model, n, loss_fn=loss, zero_grads=True, slack=2.0, perturb=k == "graph_perturb", **cfg) for k in ("graph", "graph_perturb")}
    host = SingleVolumeRenderer(dict(cfg, perturb=True)).train()

    def host_step():
        model.zero_grad(set_to_none=True)
        loss(host.render(model, o, d, rays_h_appear=codes)["rendered"]).backward()

    arms = dict(graph=lambda: frames["graph"].step(o, d, codes), graph_perturb=lambda: frames["graph_perturb"].step(o, d, codes), host_perturb=host_step)
    for fn in arms.values():
        for _ in range(args.warmup):
            fn()
    for f in frames.values():
        assert f.check(retry=False), "arena overflow after the warm-up"
    torch.cuda.synchronize()
    res = {k: [] for k in arms}
    for r in range(args.rounds):
        line = {}
        order = list(arms.items())
        for k, fn in (order if r % 2 == 0 else order[::-1]):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            for _ in range(args.steps):
                fn()
            b.record()
            torch.cuda.synchronize()
            line[k] = a.elapsed_time(b) / args.steps
            res[k].append(line[k])
        print(json.dumps(dict(workload=name, round=r, ms_per_step=line)), flush=True)
    out = dict(workload=name, rays=n, captures={k: f.captures for k, f in frames.items()}, median_ms={k: statistics.median(v) for k, v in res.items()})
    del frames
    gc.collect()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--only", choices=["camera", "lidar", "frame800"], default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perturb_step.py needs a CUDA device")
    dev = torch.device("cuda:0")
    out = []
    if args.only in (None, "camera"):
        out.append(run("cfg3 street 8192 camera rays", lambda: street(dev, False), args))
    if args.only in (None, "lidar"):
        out.append(run("cfg3 street 8192 LiDAR rays", lambda: street(dev, True), args))
    if args.only in (None, "frame800"):
        out.append(run("800x600 frame", lambda: frame800(dev), args))
    summary = dict(summary=out, gpu=gpu_info())
    print(json.dumps(summary), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
