"""The shipped StreetSurf camera encoding (ngp, 32 Mi parameters, 2^20 hash map, no level cap: 17 levels on the cfg3 street box) on the
48-column kernels: what fusing it buys, and what the wider tile costs against the 16-level form.  Arms, alternated in rounds in one
process, each timed with CUDA events around whole steps (forward + loss + backward):
  module17   the 17-level model as it runs by default (max_fused_levels=16): the unfused module path
  host17     the 17-level model with max_fused_levels=24: the host-sized fused step (SingleVolumeRenderer.render + backward)
  graph17    the same model in the one-launch graph step (StaticFrame)
  host16 / graph16   the 16-level form of the model (bench_cfg3's cfg3 workload) on the same rays, as the reference point
  graph17_codes / graph16_codes   (camera rays) the graph step with the appearance-code gradient (StaticFrame(h_appear_grad=True)), as a
             camera model trains: the ray-tiled code form of the colour backward (k_color_rad_bwd<true, ., NF>) and the per-ray code sums
The other arms pass constant codes (zeros, no gradient) and no pose.  bench_cfg3.build_model passes no surface keywords, so the 17-level model
gets the option as the attribute LoTDSDF(max_fused_levels=24) sets; the module arm sets it back to 16 for its step.
Workloads: 8192 camera rays (rgb + normals + appearance codes) and 8192 LiDAR rays.  Prints one JSON line per round and workload and a
summary with the GPU name, power limit and SM clocks read in the same run; then, in a separate torch.profiler run, the per-kernel CUDA
times of one host-sized camera step at 16 and at 17 levels.  `--out FILE` also writes the summary there.

    python profiles/wide_levels_step.py --steps 20 --warmup 5 --rounds 4
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


def models(dev):
    import bench_cfg3 as C
    m17 = C.build_model(dev, max_num_levels=None).train()
    m17.implicit_surface.max_fused_levels = 24          # LoTDSDF(max_fused_levels=24), set after bench_cfg3 built it
    m16 = C.build_model(dev).train()
    assert m17.implicit_surface.encoding.meta.n_pseudo_levels == 17 and m16.implicit_surface.encoding.meta.n_pseudo_levels == 16
    assert m17._color_fusable() and m16._color_fusable()
    return m17, m16


def rays(dev, lidar, m):
    import bench_cfg3 as C
    if lidar:
        o, d = C.lidar_rays(1, C.N_LIDAR)
        return o.to(dev), d.to(dev), None, C.loss_lidar, dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True)
    o, d = C.camera_rays(3, C.N_CAM)
    na = m.radiance_net.blocks.layers[0].in_features - 22 - m.implicit_surface.encoding.out_features
    return o.to(dev), d.to(dev), torch.zeros(o.shape[0], na, device=dev), C.loss_cam, dict(near=C.NEAR, far=C.FAR)


def run(name, lidar, m17, m16, args):
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.renderer import SingleVolumeRenderer
    o, d, codes, loss, cfg = rays(m17.device, lidar, m17)
    n = o.shape[0]
    gc.collect()
    frames = {"graph17": StaticFrame(m17, n, loss_fn=loss, zero_grads=True, slack=2.0, **cfg),
              "graph16": StaticFrame(m16, n, loss_fn=loss, zero_grads=True, slack=2.0, **cfg)}
    if not lidar:
        frames.update(graph17_codes=StaticFrame(m17, n, loss_fn=loss, zero_grads=True, slack=2.0, h_appear_grad=True, **cfg),
                      graph16_codes=StaticFrame(m16, n, loss_fn=loss, zero_grads=True, slack=2.0, h_appear_grad=True, **cfg))
    r = SingleVolumeRenderer(cfg).train()

    def host(m, fused):
        def step():
            s = m.implicit_surface
            s.max_fused_levels = 24 if fused else 16
            m.zero_grad(set_to_none=True)
            loss(r.render(m, o, d, rays_h_appear=codes)["rendered"]).backward()
            s.max_fused_levels = 24
        return step

    arms = dict(module17=host(m17, False), host17=host(m17, True), graph17=lambda: frames["graph17"].step(o, d, codes),
                host16=host(m16, True), graph16=lambda: frames["graph16"].step(o, d, codes))
    if not lidar:
        arms.update(graph17_codes=lambda: frames["graph17_codes"].step(o, d, codes), graph16_codes=lambda: frames["graph16_codes"].step(o, d, codes))
    for fn in arms.values():
        for _ in range(args.warmup):
            fn()
    for f in frames.values():
        assert f.check(retry=False), "arena overflow after the warm-up"
    torch.cuda.synchronize()
    res = {k: [] for k in arms}
    for rd in range(args.rounds):
        line = {}
        order = list(arms.items())
        for k, fn in (order if rd % 2 == 0 else order[::-1]):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            for _ in range(args.steps):
                fn()
            b.record()
            torch.cuda.synchronize()
            line[k] = a.elapsed_time(b) / args.steps
            res[k].append(line[k])
        print(json.dumps(dict(workload=name, round=rd, ms_per_step=line)), flush=True)
    out = dict(workload=name, rays=n, captures={k: f.captures for k, f in frames.items()}, median_ms={k: statistics.median(v) for k, v in res.items()})
    del frames
    gc.collect()
    torch.cuda.empty_cache()
    return out


def kernel_times(m17, m16):
    """per-kernel CUDA time (ms) of one host-sized camera step at 17 and at 16 levels (torch.profiler, after a warm-up step)"""
    from torch.profiler import ProfilerActivity, profile
    from neuralsim_b200.renderer import SingleVolumeRenderer
    out = {}
    for tag, m in (("17", m17), ("16", m16)):
        o, d, codes, loss, cfg = rays(m.device, False, m)
        r = SingleVolumeRenderer(cfg).train()

        def step():
            m.zero_grad(set_to_none=True)
            loss(r.render(m, o, d, rays_h_appear=codes)["rendered"]).backward()
        step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as p:
            step()
            torch.cuda.synchronize()
        times = {}
        for e in p.key_averages():
            if e.device_type.name == "CUDA" and e.key.startswith("void nsb::k_"):
                times[e.key.split("(")[0].replace("void nsb::", "")] = round(e.device_time_total / 1000.0, 4)
        out[tag] = dict(sorted(times.items(), key=lambda kv: -kv[1]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("wide_levels_step.py needs a CUDA device")
    dev = torch.device("cuda:0")
    m17, m16 = models(dev)
    out = [run("cfg3 street 8192 camera rays", False, m17, m16, args), run("cfg3 street 8192 LiDAR rays", True, m17, m16, args)]
    summary = dict(summary=out, gpu=gpu_info())
    print(json.dumps(summary), flush=True)
    summary["kernel_ms_camera_step"] = kernel_times(m17, m16)
    print(json.dumps(dict(kernel_ms_camera_step=summary["kernel_ms_camera_step"])), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
