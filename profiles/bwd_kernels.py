"""Device time per step of the backward and forward wgmma kernels in the bench workload (cfg2: one 800x600 frame, fwd+bwd), with
torch.profiler (CUPTI) over 5 kernel-by-kernel StaticFrame steps, plus the point counts those kernels ran over.
    python profiles/bwd_kernels.py [--steps 5]
Prints one JSON line: ms per step of each kernel, the kept samples (colour kernels) and the samples with a non-zero sdf cotangent
(k_sdf_bwd_tc) per step, and the GPU name, power limit and maximum SM clock the numbers were taken at."""
import argparse
import json
import os
import subprocess
import sys

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from neuralsim_b200.graphics.neus_static import CNT_SLOTS, StaticFrame  # noqa: E402

KERNELS = ("k_color_rad_bwd", "k_color_sdf_bwd", "k_sdf_bwd_tc", "k_color_fwd", "k_fused_sdf_tc")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa: BLE001 -- the numbers stand without it, but say why it is missing
        return dict(gpu=torch.cuda.get_device_name(0), power_limit=f"unknown ({e})")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    model = bench.build_model(dev).train()
    flat, _ = bench.flat_grad_views(model)
    o, d = bench.pinhole_rays(bench.H, bench.W, bench.orbit(0, bench.N_VIEWS))
    o, d = o.to(dev), d.to(dev)
    frame = StaticFrame(model, o.shape[0], loss_fn=bench.loss_of, near=0.01, use_graph=False, pre_hook=flat.zero_)
    for _ in range(3):                              # sizes the arenas, then warms up
        frame.step(o, d, None)
    torch.cuda.synchronize()
    kept = nonzero = 0
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            frame.step(o, d, None)
            torch.cuda.synchronize()
            c = frame.cnt.tolist()
            kept += c[CNT_SLOTS["kept"]]
            nonzero += c[CNT_SLOTS["nonzero"]]
    us = {k: 0.0 for k in KERNELS}
    calls = {k: 0 for k in KERNELS}
    for e in prof.key_averages():
        for k in KERNELS:
            if k in e.key:
                us[k] += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                calls[k] += e.count
    line = dict(ms_per_step={k: round(us[k] / 1e3 / args.steps, 4) for k in KERNELS},
                launches_per_step={k: calls[k] / args.steps for k in KERNELS},
                colour_bwd_ms_per_step=round((us["k_color_rad_bwd"] + us["k_color_sdf_bwd"]) / 1e3 / args.steps, 4),
                kept_per_step=kept / args.steps, nonzero_cotangent_per_step=nonzero / args.steps, steps=args.steps, **gpu_info())
    print(json.dumps(line))


if __name__ == "__main__":
    main()
