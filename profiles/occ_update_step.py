"""The occupancy grid's update from the network: host-sized (OccGridEma.step: nonzero() host reads, torch sampling, host-sized SDF queries)
against one replay of fields/occ_update.py:OccGridUpdate.  Two measurements per workload, arms alternated in rounds in one process:
  update   one update (the shipped update_from_net_cfg: 4 iterations of 2^20 points), CUDA events around it, median over --reps, per phase
  loop     160 iterations of 8192-ray StaticFrame steps with an update every 16 (steady phase), host clock around the loop ending in a
           device synchronise: wall ms per iteration -- what the host reads of the host-sized update cost a loop of graph steps
Workloads: the cfg3 street model (bench_cfg3.build_model, 40 x 150 x 15 grid) with camera rays, and bench.py's CFG model (64^3 grid).
Prints one JSON line per measurement and a summary with the GPU name, power limit and SM clocks read in the same run; `--out FILE` also
writes the summary there.

    python profiles/occ_update_step.py --rounds 3 --reps 10
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

N_RAYS, ITERS = 8192, 160


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def workload(name, dev):
    import bench
    import bench_cfg3 as C
    if name == "cfg3":
        model = C.build_model(dev).train()
        views = [C.camera_rays(k, N_RAYS) for k in range(8)]
        return model, [(o.to(dev), d.to(dev)) for o, d in views], C.loss_cam, dict(near=C.NEAR, far=C.FAR)
    torch.manual_seed(0)
    model = bench.build_model(dev, collect_samples=True).train()
    views = []
    for k in range(8):
        o, d = bench.pinhole_rays(bench.H, bench.W, bench.orbit(k, 8))
        sel = torch.randperm(o.shape[0], generator=torch.Generator().manual_seed(k))[:N_RAYS]
        views.append((o[sel].to(dev), d[sel].to(dev)))
    return model, views, bench.loss_of, dict(near=0.01)


def time_update(model, upd, it, reps):
    occ = model.accel.occ
    occ.net_update = upd
    ts = []
    for _ in range(reps + 2):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        assert occ.step(it, model.query_sdf)
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    occ.net_update = None
    return statistics.median(ts[2:])


def time_loop(model, frame, upd, views):
    occ = model.accel.occ
    occ.net_update = upd
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for it in range(1, ITERS + 1):
        model.training_before_per_step(it)
        o, d = views[it % len(views)]
        frame.step(o, d)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / ITERS
    occ.net_update = None
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("occ_update_step.py: needs a CUDA device")
    from neuralsim_b200.fields import OccGridUpdate
    from neuralsim_b200.graphics.neus_static import StaticFrame
    dev = torch.device("cuda")
    summary = dict(gpu=gpu_info(), rays=N_RAYS, iterations=ITERS)
    for name in ("cfg3", "cfg64"):
        model, views, loss_fn, rc = workload(name, dev)
        occ = model.accel.occ
        occ.update_from_net_cfg = dict(num_steps=4, num_pts=2 ** 20)
        occ.n_steps_between_update, occ.n_steps_warmup = 16, 0
        upd = OccGridUpdate(model)
        occ.net_update = None
        frame = StaticFrame(model, N_RAYS, loss_fn=loss_fn, zero_grads=True, **rc)
        frame.step(*views[0])
        res = {"update_host_warmup": [], "update_graph_warmup": [], "update_host": [], "update_graph": [], "loop_host": [], "loop_graph": []}
        occ.n_steps_warmup = 10 ** 9
        time_update(model, upd, 16, 1)                             # capture
        for r in range(args.rounds):
            res["update_host_warmup"].append(time_update(model, None, 16, args.reps))
            res["update_graph_warmup"].append(time_update(model, upd, 16, args.reps))
        occ.n_steps_warmup = 0
        for r in range(args.rounds):
            res["update_host"].append(time_update(model, None, 16, args.reps))
            res["update_graph"].append(time_update(model, upd, 16, args.reps))
            res["loop_host"].append(time_loop(model, frame, None, views))
            res["loop_graph"].append(time_loop(model, frame, upd, views))
            print(json.dumps(dict(workload=name, round=r, **{k: round(v[-1], 3) for k, v in res.items()})), flush=True)
        frame.check(retry=False)
        summary[name] = {k: round(statistics.median(v), 3) for k, v in res.items()}
        summary[name]["n_occupied"] = int(occ.occ_grid.sum())
        del frame, upd, model
        torch.cuda.empty_cache()
    summary["gpu_after"] = gpu_info()
    print(json.dumps(summary), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
