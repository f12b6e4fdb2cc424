"""The shipped LiDAR-only StreetSurf configuration (lidaronly_filterobj.240219.yaml: a 12-level LoTD table of 32 Mi target parameters,
log2 hashmap 20, no radiance net, num_coarse 256, num_fine [8, 8, 8], march step 0.05) on the cfg3 street box, one training step on
8192 LiDAR rays (bench_cfg3.lidar_rays).  Three arms, one JSON line each per round:

  parent:host   another checkout (--parent ROOT, its library built) -- a checkout whose wgmma kernels take only 16-level tables runs this
                model on the module path (LoTD forward_dydx -> decoder -> autograd.grad -> backward_dydx)
  built:host    this checkout, the host-sized fused step (SingleVolumeRenderer + loss + backward)
  built:graph   this checkout, the one-launch graph step (StaticFrame)

Each checkout runs in its own process; rounds alternate the order.  The GPU name, power limit and SM clocks are read in the same run.
Usage: python profiles/lidar_only_shipped_step.py --parent ROOT [--steps 30] [--warmup 8] [--rounds 3] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RAYS = 8192


def _model(dev):
    import torch
    import bench_cfg3 as C
    from neuralsim_b200.fields import LoTDNeuSModel
    gen = torch.Generator(device=dev).manual_seed(42)
    m = LoTDNeuSModel(
        surface_cfg=dict(aabb=C.AABB, sdf_scale=C.SDF_SCALE, encoding_cfg=dict(lotd_use_cuboid=True, lotd_auto_compute_cfg=dict(
            type="ngp", target_num_params=32 * 2 ** 20, min_res=16, n_feats=2, log2_hashmap_size=20, max_num_levels=12),
            param_init_cfg=dict(type="uniform_to_type", bound=2.0e-3))),
        radiance_cfg=False, var_ctrl_cfg=dict(ln_inv_s_init=0.5298, ln_inv_s_factor=10.0),
        accel_cfg=dict(vox_size=1.0, occ_val_fn_cfg=dict(type="sdf", inv_s=256.0), occ_thre=0.3, ema_decay=0.95, update_from_samples_cfg=None),
        ray_query_cfg=dict(query_mode="march_occ_multi_upsample_compressed", query_param=dict(
            nablas_has_grad=True, num_coarse=256, num_fine=[8, 8, 8], coarse_step_cfg=dict(step_mode="linear"),
            march_cfg=dict(step_size=0.05, max_steps=4096), upsample_inv_s=64.0, upsample_inv_s_factors=[1, 4, 16], upsample_use_estimate_alpha=False)),
        device=dev, generator=gen)
    assert m.implicit_surface.encoding.meta.n_pseudo_levels == 12
    return C.install_plane(m, C.ROAD_Z).train()


def _time(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    ms.sort()
    return dict(mean_ms=sum(ms) / len(ms), median_ms=ms[len(ms) // 2], min_ms=ms[0], max_ms=ms[-1])


def worker(args):
    sys.path.insert(0, args.root)
    import torch
    import bench_cfg3 as C
    from neuralsim_b200.renderer import SingleVolumeRenderer
    from neuralsim_b200.graphics.neus_static import StaticFrame
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    model = _model(dev)
    lo, ld = C.lidar_rays(1, RAYS)
    lo, ld = lo.to(dev), ld.to(dev)
    for mode in args.modes.split(","):
        if mode == "host":
            r = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True)).train()

            def step():
                model.zero_grad(set_to_none=False)
                C.loss_lidar(r.render(model, lo, ld)["rendered"]).backward()
        else:
            fr = StaticFrame(model, RAYS, loss_fn=C.loss_lidar, near=C.NEAR, far=C.FAR, with_rgb=False, slack=1.5, zero_grads=True)

            def step():
                fr.step(lo, ld, None)
        t = _time(step, args.steps, args.warmup)
        print(json.dumps(dict(arm=f"{args.variant}:{mode}", rays=RAYS, fused=bool(model._geometry_fusable()), **t)), flush=True)


def _run(cmd):
    p = subprocess.run(cmd, capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError(f"{' '.join(cmd)} failed:\n{p.stdout}\n{p.stderr[-4000:]}")
    return [json.loads(l) for l in p.stdout.splitlines() if l.startswith("{")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", required=False)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", action="store_true")
    ap.add_argument("--root", default=ROOT)
    ap.add_argument("--modes", default="host")
    ap.add_argument("--variant", default="")
    args = ap.parse_args()
    if args.worker:
        worker(args)
        return
    q = lambda: subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                               capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=q())), flush=True)
    me = os.path.abspath(__file__)
    configs = [("built", ROOT, "host,graph")]
    if args.parent:
        configs.append(("parent", os.path.abspath(args.parent), "host"))
    results = []
    for rnd in range(args.rounds):
        for name, root, modes in (configs if rnd % 2 == 0 else configs[::-1]):
            for r in _run([sys.executable, me, "--worker", "--root", root, "--modes", modes, "--variant", name,
                           "--steps", str(args.steps), "--warmup", str(args.warmup)]):
                r["round"] = rnd
                results.append(r)
                print(json.dumps(r), flush=True)
    summary = {}
    for r in results:
        summary.setdefault(r["arm"], []).append(r["median_ms"])
    print(json.dumps(dict(summary={k: dict(medians_ms=v, best_median_ms=min(v)) for k, v in summary.items()}, gpu_after=q())), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "lidar_only_shipped_step.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
