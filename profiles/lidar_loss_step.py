"""The StreetSurf LiDAR loss (neuralsim_b200/loss/lidar.py: l1 depth + neus_unisim line of sight, discard_toofar 80, the median outlier
discard) on the cfg3 model (bench_cfg3.py: cuboid LoTD at 16 levels) with 8192 LiDAR rays per step (with_rgb=False, with_normal=True, as
the LiDAR batches of the shipped configurations train).  Arms, alternated in rounds in one process, each timed with CUDA events around whole
steps (forward + loss + backward, ending in a device synchronise):
  graph        the one-launch graph step, StaticFrame(loss_on_ret=True) with the fused loss (LidarLoss.set_step before each replay)
  host-fused   the host-sized step (SingleVolumeRenderer.render, return_buffer=True) with the fused loss
  host-torch   the host-sized step with the reference's torch formulation of the loss (sort, repeat_interleave, packed sums)
Also reports this library's launches per step (nsb_launch_count; a graph replay launches none from the host) and whether the step makes a
host sync (torch's sync debug mode, the host-sized arms' render included).  Prints one JSON line per round and a summary line with the GPU
name, power limit and SM clocks read in the same run.

    python profiles/lidar_loss_step.py --steps 20 --warmup 5 --rounds 3
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CFG = dict(discard_outliers=0, discard_outliers_median=100.0, discard_toofar=80.0, depth=dict(w=0.05, fn_type="l1"),
           line_of_sight=dict(w=0.1, fn_type="neus_unisim", fn_param=dict(epsilon_anneal=dict(type="milestones", milestones=[5000, 10000],
                                                                                               vals=[1.5, 0.75, 0.5]))))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def torch_lidar(ret, ranges, it):
    """app/loss/lidar.py LidarLoss.forward at CFG, in plain torch"""
    from neuralsim_b200.loss.lidar import anneal_milestones
    depth_pred = ret["rendered"]["depth_volume"]
    gt = ranges.view(depth_pred.shape)
    mask = gt <= 80.0
    err = (depth_pred - gt).abs() * mask
    sv, _ = torch.sort(err.data)
    mask[err > sv[depth_pred.numel() // 2] * 100.0] = False
    out = {"lidar_loss.depth": 0.05 * ((depth_pred - gt).abs() * mask).mean()}
    vb = ret["volume_buffer"]
    if vb["type"] == "packed":
        rih, t, vw, pi = vb["rays_inds_hit"], vb["t"], vb["vw"], vb["pack_infos_hit"]
        gt_ex = torch.repeat_interleave(gt[rih], pi[:, 1], dim=0)
        sel = (t - gt_ex).abs() > anneal_milestones(it, [5000, 10000], [1.5, 0.75, 0.5])
        per = torch.zeros(pi.shape[0], device=vw.device).index_add(0, torch.repeat_interleave(torch.arange(pi.shape[0], device=vw.device), pi[:, 1]),
                                                                   sel * vw ** 2)
        out["lidar_loss.los.empty"] = 0.1 * (per * mask[rih]).mean()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lidar_loss_step.py needs a CUDA device")
    import bench_cfg3 as C
    from neuralsim_b200 import _lib as L
    from neuralsim_b200.graphics.neus_static import StaticFrame
    from neuralsim_b200.loss import LidarLoss
    from neuralsim_b200.renderer import SingleVolumeRenderer
    dev = torch.device("cuda:0")
    model = C.build_model(dev).train()
    cfg = dict(near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True)
    batches = []
    for k in range(4):
        lo, ld = (x.to(dev) for x in C.lidar_rays(k, C.N_LIDAR))
        with torch.no_grad():
            d = SingleVolumeRenderer(cfg).train().render(model, lo, ld)["rendered"]["depth_volume"]
        g = torch.Generator(device=dev).manual_seed(k)
        r = (d * (1 + 0.05 * torch.randn(d.shape, device=dev, generator=g))).clamp_min(0.5)
        r[::23] = 120.0
        batches.append((lo, ld, r.contiguous()))
    lidar = LidarLoss(**CFG)
    terms = {}

    def loss_fn(ret):
        terms.update(lidar(None, ret))
        return sum(terms.values())
    renderer = SingleVolumeRenderer(cfg).train()

    def host(b, it, fused):
        lo, ld, r = b
        ret = renderer.render(model, lo, ld, return_buffer=True)
        t = lidar(None, ret, None, {"ranges": r}, it=it) if fused else torch_lidar(ret, r, it)
        sum(t.values()).backward()

    frame = StaticFrame(model, C.N_LIDAR, loss_fn=loss_fn, loss_on_ret=True, near=C.NEAR, far=C.FAR, with_rgb=False, with_normal=True, zero_grads=True)

    def graph(b, it):
        lidar.set_step(b[2], it)
        frame.step(b[0], b[1])

    arms = {"graph": lambda b, it: graph(b, it), "host-fused": lambda b, it: host(b, it, True), "host-torch": lambda b, it: host(b, it, False)}
    info = {}
    for name, fn in arms.items():
        for i in range(args.warmup):
            model.zero_grad(set_to_none=name != "graph")
            fn(batches[i % 4], 100 * i)
        torch.cuda.synchronize()
        n0 = L.launch_count()
        fn(batches[0], 0)
        torch.cuda.synchronize()
        launches = L.launch_count() - n0
        torch.cuda.set_sync_debug_mode("error")
        try:
            fn(batches[1], 0)
            syncs = "none"
        except RuntimeError as e:
            syncs = f"yes ({str(e).splitlines()[0][:80]})"
        finally:
            torch.cuda.set_sync_debug_mode("default")
        torch.cuda.synchronize()
        info[name] = dict(nsb_launches_per_step=launches, host_sync=syncs)
    rounds = {k: [] for k in arms}
    for rd in range(args.rounds):
        row = {}
        for name, fn in arms.items():
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for i in range(args.steps):
                if name != "graph":
                    model.zero_grad(set_to_none=True)
                fn(batches[i % 4], 100 * i)
            b.record()
            torch.cuda.synchronize()
            row[name] = a.elapsed_time(b) / args.steps
            rounds[name].append(row[name])
        print(json.dumps(dict(round=rd, ms_per_step=row)))
    print(json.dumps(dict(gpu=gpu_info(), steps=args.steps, rounds=args.rounds, n_rays=C.N_LIDAR, captures=frame.captures,
                          median_ms_per_step={k: statistics.median(v) for k, v in rounds.items()}, **{k: info[k] for k in info})))


if __name__ == "__main__":
    main()
