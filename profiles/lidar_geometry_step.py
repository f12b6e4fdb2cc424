"""LiDAR-ray steps on the cfg3 street model (bench_cfg3.py) with the geometry-only colour query (k_color_fwd<false>): one JSON line per arm.

  (a) a geometry-only cfg3 model (radiance_cfg=False, the LiDAR-only StreetSurf configuration) at 8192 rays and at one 64 x 2048 sweep
      (131 072 rays): the host-sized step (SingleVolumeRenderer + loss + backward), the graph step (StaticFrame) and the same model on the
      module path (forward_sdf_nablas + autograd); with the library as built and, alternated with it, another build of this checkout's
      library (--alt-lib PATH, geometry-only arms only; DESIGN.md §6's 3-CTA residency was such a build);
  (b) the cfg3 colour model's LiDAR arm (8192 rays, host-sized and graph) against another checkout (--parent ROOT, its library built),
      alternated with this one; the rendered buffers of one fixed batch are compared bit for bit;
  (c) torch.profiler runs (a process per library) with the device time per step of each colour kernel.

Each configuration runs in its own process (one library per process); rounds alternate them.  Prints the GPU name, power limit and SM clock.
Usage: python profiles/lidar_geometry_step.py [--parent ROOT] [--alt-lib PATH] [--steps 30] [--warmup 8] [--rounds 3] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------------------ worker (one library)
def _geo_model(dev):
    import bench_cfg3 as C
    from neuralsim_b200.fields import LoTDNeuSModel
    gen = __import__("torch").Generator(device=dev).manual_seed(42)
    m = LoTDNeuSModel(
        surface_cfg=dict(aabb=C.AABB, sdf_scale=C.SDF_SCALE, encoding_cfg=dict(lotd_use_cuboid=True, lotd_auto_compute_cfg=dict(
            type="ngp", target_num_params=32 * 2 ** 20, min_res=16, n_feats=2, log2_hashmap_size=20, max_num_levels=16),
            param_init_cfg=dict(type="uniform_to_type", bound=2.0e-3))),
        radiance_cfg=False, var_ctrl_cfg=dict(ln_inv_s_init=0.5298, ln_inv_s_factor=10.0),
        accel_cfg=dict(vox_size=1.0, occ_val_fn_cfg=dict(type="sdf", inv_s=256.0), occ_thre=0.3, ema_decay=0.95, update_from_samples_cfg=None),
        ray_query_cfg=dict(query_mode="march_occ_multi_upsample_compressed", query_param=dict(
            nablas_has_grad=True, num_coarse=128, num_fine=[8, 8, 32], coarse_step_cfg=dict(step_mode="linear"),
            march_cfg=dict(step_size=0.2, max_steps=4096), upsample_inv_s=64.0, upsample_inv_s_factors=[1, 4, 16], upsample_use_estimate_alpha=False)),
        device=dev, generator=gen)
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
    import neuralsim_b200._lib as L
    if args.lib:
        L.LIB_PATH = args.lib
    import bench_cfg3 as C
    from neuralsim_b200.renderer import SingleVolumeRenderer
    from neuralsim_b200.graphics.neus_static import StaticFrame
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    res = []
    arms = args.arms.split(",")
    sizes = [8192, 131072]
    for arm in arms:
        kind, mode = arm.split(":")            # geo|geo_module|colour : host|graph
        model = C.build_model(dev).train() if kind == "colour" else _geo_model(dev)
        if kind == "geo_module":
            model._geometry_fusable = lambda: False
        for n in (sizes if kind != "colour" else [8192]):
            lo, ld = C.lidar_rays(1, n)
            lo, ld = lo.to(dev), ld.to(dev)
            if mode == "host":
                r = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True)).train()

                def step():
                    model.zero_grad(set_to_none=False)
                    C.loss_lidar(r.render(model, lo, ld)["rendered"]).backward()
            else:
                fr = StaticFrame(model, n, loss_fn=C.loss_lidar, near=C.NEAR, far=C.FAR, with_rgb=False, slack=1.5, zero_grads=True)

                def step():
                    fr.step(lo, ld, None)
            t = _time(step, args.steps, args.warmup)
            out = dict(variant=args.variant, arm=arm, rays=n, **t)
            if args.dump and mode == "host" and n == 8192:
                with torch.no_grad():
                    rend = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True)).train().render(model, lo, ld)["rendered"]
                torch.save({k: v.detach().cpu() for k, v in rend.items()}, os.path.join(args.dump, f"{args.variant}_{kind}.pt"))
            res.append(out)
            print(json.dumps(out), flush=True)
            del step
        del model
        torch.cuda.empty_cache()
    return res


def profile_worker(args):
    """(c): device time per step of every colour kernel: colour model (camera + LiDAR arm) and geometry-only model"""
    sys.path.insert(0, args.root)
    import torch
    import neuralsim_b200._lib as L
    if args.lib:
        L.LIB_PATH = args.lib
    from torch.profiler import ProfilerActivity, profile
    import bench_cfg3 as C
    from neuralsim_b200.renderer import SingleVolumeRenderer
    dev = torch.device("cuda", 0)
    out = {}
    for kind in (("colour", "geo") if args.variant != "parent" else ("colour",)):
        model = C.build_model(dev).train() if kind == "colour" else _geo_model(dev)
        (co, cd), (lo, ld) = C.make_views(1)
        co, cd, lo, ld = co.to(dev), cd.to(dev), lo.to(dev), ld.to(dev)
        ha = torch.zeros(co.shape[0], 4, device=dev)
        rc = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR)).train()
        rl = SingleVolumeRenderer(dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True)).train()

        def step():
            model.zero_grad(set_to_none=False)
            loss = C.loss_lidar(rl.render(model, lo, ld)["rendered"])
            if kind == "colour":
                loss = loss + C.loss_cam(rc.render(model, co, cd, rays_h_appear=ha)["rendered"])
            loss.backward()
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                step()
            torch.cuda.synchronize()
        for e in prof.key_averages():
            if "k_color" in e.key:
                dt = getattr(e, "device_time_total", None)
                if dt is None:
                    dt = e.cuda_time_total
                out[f"{kind}:{e.key}"] = dict(ms_per_step=dt / 1000.0 / 5, launches_per_step=e.count / 5)
        del model
        torch.cuda.empty_cache()
    print(json.dumps(dict(profile=args.variant, kernels=out)), flush=True)


# ------------------------------------------------------------------------------------------------------------ driver
def _run(cmd):
    p = subprocess.run(cmd, capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError(f"{' '.join(cmd)} failed:\n{p.stdout}\n{p.stderr[-4000:]}")
    return [json.loads(l) for l in p.stdout.splitlines() if l.startswith("{")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default=None)
    ap.add_argument("--alt-lib", default=None)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    # worker options
    ap.add_argument("--worker", action="store_true")
    ap.add_argument("--profile-worker", action="store_true")
    ap.add_argument("--root", default=ROOT)
    ap.add_argument("--lib", default=None)
    ap.add_argument("--arms", default="")
    ap.add_argument("--variant", default="")
    ap.add_argument("--dump", default=None)
    args = ap.parse_args()
    if args.worker:
        worker(args)
        return
    if args.profile_worker:
        profile_worker(args)
        return
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps(dict(gpu=q.stdout.strip())), flush=True)
    tmp = tempfile.mkdtemp(prefix="nsb_lidar_geo_")
    me = os.path.abspath(__file__)
    common = ["--steps", str(args.steps), "--warmup", str(args.warmup), "--dump", tmp]
    configs = [("built", ROOT, None, "geo:host,geo:graph,geo_module:host,colour:host,colour:graph")]
    if args.alt_lib:
        configs.append(("alt", ROOT, os.path.abspath(args.alt_lib), "geo:host,geo:graph"))
    if args.parent:
        configs.append(("parent", os.path.abspath(args.parent), None, "colour:host,colour:graph"))
    results = []
    for rnd in range(args.rounds):
        for name, root, lib, arms in (configs if rnd % 2 == 0 else configs[::-1]):
            cmd = [sys.executable, me, "--worker", "--root", root, "--arms", arms, "--variant", name, *common]
            if lib:
                cmd += ["--lib", lib]
            for r in _run(cmd):
                r["round"] = rnd
                results.append(r)
                print(json.dumps(r), flush=True)
    if args.parent:
        import torch
        a, b = torch.load(os.path.join(tmp, "built_colour.pt")), torch.load(os.path.join(tmp, "parent_colour.pt"))
        print(json.dumps(dict(colour_lidar_bit_equal_to_parent={k: bool(torch.equal(a[k], b[k])) for k in b} | {"same_keys": set(a) == set(b)})), flush=True)
    for name, root, lib, _arms in configs:
        cmd = [sys.executable, me, "--profile-worker", "--root", root, "--variant", name] + (["--lib", lib] if lib else [])
        for r in _run(cmd):
            print(json.dumps(r), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "lidar_geometry_step.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
