"""Kernel-time table of one bench step with torch.profiler (CUPTI); cheaper than an ncu launch list for iterating.
    python profiles/torch_profile_step.py > torch_prof.txt
    python profiles/torch_profile_step.py --static [--steps 5]
--static profiles the bench's graph step launched kernel by kernel (StaticFrame, use_graph=False: the same launches the graph replays)
and prints one JSON line: device ms per step and launches per step of every kernel, the launch count per step, and the GPU name,
power limit and maximum SM clock the numbers were taken at."""
import argparse
import json
import os
import sys

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench  # noqa: E402
from bwd_kernels import gpu_info  # noqa: E402
from neuralsim_b200 import _lib  # noqa: E402
from neuralsim_b200.renderer import SingleVolumeRenderer  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--static", action="store_true")
ap.add_argument("--steps", type=int, default=5)
args = ap.parse_args()

dev = torch.device("cuda:0")
model = bench.build_model(dev).train()
r = SingleVolumeRenderer(dict(near=0.01)).train()
flat, params = bench.flat_grad_views(model)
o, d = bench.pinhole_rays(bench.H, bench.W, bench.orbit(0, bench.N_VIEWS if args.static else 8))
o, d = o.to(dev), d.to(dev)
CH = int(os.environ.get("CHUNK", 480000))
ha = torch.zeros(CH, 4, device=dev)
frame = None
if args.static:
    from neuralsim_b200.graphics.neus_static import StaticFrame
    frame = StaticFrame(model, o.shape[0], loss_fn=bench.loss_of, near=0.01, use_graph=False, pre_hook=flat.zero_)


def step():
    if frame is not None:
        frame.step(o, d, None)
        return
    flat.zero_()
    for s in range(0, o.shape[0], CH):
        e = min(s + CH, o.shape[0])
        out = r.render(model, o[s:e], d[s:e], rays_h_appear=ha[:e - s])["rendered"]
        loss = bench.loss_of(out) * ((e - s) / o.shape[0])
        if loss.requires_grad:
            loss.backward()


for _ in range(3):
    step()
torch.cuda.synchronize()
if not args.static:
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    print(prof.key_averages().table(sort_by="self_cuda_time_total", row_limit=45, max_name_column_width=70))
    sys.exit(0)

l0 = _lib.launch_count()
step()
torch.cuda.synchronize()
launches = _lib.launch_count() - l0
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(args.steps):
        step()
    torch.cuda.synchronize()
rows = {}
for e in prof.key_averages():
    us = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0.0)
    if us > 0:
        name = e.key.split("(")[0].replace("void ", "").split("<")[0].strip()
        rt = rows.setdefault(name, [0.0, 0])
        rt[0] += us / 1e3 / args.steps
        rt[1] += e.count / args.steps
table = sorted(([k, round(v[0], 4), v[1]] for k, v in rows.items()), key=lambda x: -x[1])
print(json.dumps(dict(ms_per_step_total=round(sum(x[1] for x in table), 3), nsb_launches_per_step=launches, steps=args.steps,
                      kernels=table, **gpu_info())))
