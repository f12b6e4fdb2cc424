"""What the LoTD level schedule costs and saves on the cfg3 colour model (bench_cfg3.py: cuboid LoTD at 16 levels, 32 Mi parameters), on one
GPU, with the GPU's name, power limit and SM clocks read in the same run:
  graph      the one-launch graph step (StaticFrame, 8192 camera rays, loss_cam) at the encoding's max_level 2 / 6 / 10 / 15 / None: one
             capture sized at all levels, the level refilled before every replay as the schedule does; ms per step from CUDA events
             around whole replays (ending in a device synchronise)
  kernels    the host-sized step (SingleVolumeRenderer.render + backward) at the same levels with CUDA events around every launch of the
             forward gathers (the boundary SDF query fused_sdf_fwd, the up-sampling ray_upsample, the colour forward fused_color_fwd) and of
             the backward kernels: ms per step of each
             and, with --parent DIR, the same in the parent commit's tree (whose forward gathers load every level and zero the masked ones)
  bench      (with --parent DIR, a built checkout of the parent commit) `bench.py --gpus 1 --steps S --warmup W --no-cpu-baseline
             --no-ref-cuda` of this tree and of DIR alternated for --rounds rounds, and `bench.py --dump-outputs` of both, whose files
             are compared bit for bit
Prints one JSON line per part and, with --out FILE, writes them all to FILE as one JSON document.

    python profiles/lotd_anneal_step.py --steps 20 --warmup 5 [--parent ../parent --rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# --tree DIR: import the package (and bench_cfg3) from another checkout, e.g. the parent commit's, for the host-sized kernels part
TREE = os.path.abspath(sys.argv[sys.argv.index("--tree") + 1]) if "--tree" in sys.argv else ROOT
sys.path.insert(0, TREE)
LEVELS = [2, 6, 10, 15, None]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def _timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return ts


def graph_part(args):
    import bench_cfg3 as C
    from neuralsim_b200.graphics.neus_static import StaticFrame
    dev = torch.device("cuda")
    model = C.build_model(dev).train()
    enc = model.implicit_surface.encoding
    co, cd = (t.to(dev) for t in C.camera_rays(0, C.N_CAM))
    ha = torch.zeros(C.N_CAM, 4, device=dev)
    fr = StaticFrame(model, C.N_CAM, loss_fn=C.loss_cam, near=C.NEAR, far=C.FAR, zero_grads=True, slack=2.0)
    fr.step(co, cd, ha)                                    # sized and captured at all levels
    out = {}
    for ml in LEVELS:
        enc.max_level = ml
        ts = _timed(lambda: fr.step(co, cd, ha), args.steps, args.warmup)
        c = fr.counts()
        out[str(ml)] = dict(ms_median=float(np.median(ts)), ms_min=float(min(ts)), overflow=c["overflow"], kept=c["kept"], boundary=c["boundary"])
    enc.max_level = None
    assert fr.captures == 1
    return out


def kernels_part(args):
    import bench_cfg3 as C
    from neuralsim_b200 import _lib as L
    from neuralsim_b200.renderer import SingleVolumeRenderer
    dev = torch.device("cuda")
    model = C.build_model(dev).train()
    enc = model.implicit_surface.encoding
    co, cd = (t.to(dev) for t in C.camera_rays(0, C.N_CAM))
    ha = torch.zeros(C.N_CAM, 4, device=dev)
    r = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR)).train()

    def step():
        model.zero_grad(set_to_none=True)
        C.loss_cam(r.render(model, co, cd, rays_h_appear=ha)["rendered"]).backward()
    out = {}
    for ml in LEVELS:
        enc.max_level = ml
        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        L.KERNEL_TIMER.enable()
        for _ in range(args.steps):
            step()
        s = L.KERNEL_TIMER.summary()
        L.KERNEL_TIMER.disable()
        out[str(ml)] = {k: dict(ms_per_step=v["ms"] / args.steps, points_per_step=v["units"] / args.steps) for k, v in sorted(s.items())}
    enc.max_level = None
    return out


def _bench(tree, args, dump=None):
    cmd = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", str(args.bench_steps), "--warmup", str(args.bench_warmup),
           "--no-cpu-baseline", "--no-ref-cuda"]
    if dump:
        cmd = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", "2", "--warmup", "1", "--no-cpu-baseline", "--no-ref-cuda",
               "--dump-outputs", dump]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=tree, timeout=1800)
    if r.returncode != 0:
        raise RuntimeError(f"bench.py in {tree} failed:\n{r.stderr[-3000:]}")
    line = json.loads(r.stdout.strip().splitlines()[-1])
    return dict(ms_per_step=line["ms_per_step"], median_ms=line["median"]["ms_per_step"], value=line["value"], clocks=line.get("clocks"))


def bench_part(args):
    parent = os.path.abspath(args.parent)
    rounds = {"this": [], "parent": []}
    for _ in range(args.rounds):
        for name, tree in (("parent", parent), ("this", ROOT)):
            rounds[name].append(_bench(tree, args))
    with tempfile.TemporaryDirectory() as tmp:
        a, b = os.path.join(tmp, "this"), os.path.join(tmp, "parent")
        _bench(ROOT, args, dump=a)
        _bench(parent, args, dump=b)
        files = sorted(os.listdir(b))
        same = {f: bool(np.array_equal(np.load(os.path.join(a, f)), np.load(os.path.join(b, f)), equal_nan=True)) for f in files}
        assert sorted(os.listdir(a)) == files
    return dict(rounds=rounds, dump_outputs_bit_equal=same)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--parent", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--bench-steps", type=int, default=20)
    ap.add_argument("--bench-warmup", type=int, default=10)
    ap.add_argument("--parts", default="graph,kernels,bench")
    ap.add_argument("--tree", default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "lotd_anneal_step.py measures on a GPU"
    res = dict(gpu=gpu_info())
    parts = args.parts.split(",")
    if "graph" in parts:
        res["graph"] = graph_part(args)
        print(json.dumps(dict(part="graph", **res["graph"])), flush=True)
    if "kernels" in parts:
        res["kernels"] = kernels_part(args)
        print(json.dumps(dict(part="kernels", **res["kernels"])), flush=True)
    if "kernels" in parts and args.parent:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--parts", "kernels", "--tree", os.path.abspath(args.parent), "--steps", str(args.steps),
                            "--warmup", str(args.warmup)], capture_output=True, text=True, timeout=1800)
        if r.returncode != 0:
            raise RuntimeError(r.stderr[-3000:])
        res["kernels_parent"] = json.loads(r.stdout.strip().splitlines()[0])
        res["kernels_parent"].pop("part")
        print(json.dumps(dict(part="kernels_parent", **res["kernels_parent"])), flush=True)
    if "bench" in parts and args.parent:
        res["bench"] = bench_part(args)
        print(json.dumps(dict(part="bench", **res["bench"])), flush=True)
    res["gpu_after"] = gpu_info()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(dict(gpu=res["gpu"], gpu_after=res["gpu_after"])), flush=True)


if __name__ == "__main__":
    main()
